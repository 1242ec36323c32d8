"""KVzap scores and DMS eviction on one GPU: the fused kernels against the reference's path restated in torch.

Layer shape of Llama-3.1-8B / Qwen3-8B (hidden 4096, 8 kv heads, MLP width 512, bf16). The torch path is the
reference's: the module cast to the device and dtype, Linear -> GELU -> Linear, the transpose, and torch.where for the
eviction. Each call is timed with CUDA events over many launches after a warm-up, as issued from Python (`ms`, which
includes the host's call overhead) and replayed from a CUDA graph (`graph_ms`, device time; TFLOP/s come from it). The
eviction reads its count on the host, as torch.where does, so it is timed from Python only. The card's name and power
limit are read in the same run. Prints one JSON line per case.
"""
import json
import subprocess
import sys
from pathlib import Path

import torch
import torch.nn as nn

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from kvpress_b200 import native  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def timed(fn, iters):
    for _ in range(3):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def main():
    dev, dtype, hidden, H, hd = "cuda", torch.bfloat16, 4096, 8, 512
    name = card()
    torch.manual_seed(0)
    for kind in ("mlp", "linear"):
        module = (nn.Sequential(nn.Linear(hidden, hd), nn.GELU(), nn.Linear(hd, H)) if kind == "mlp"
                  else nn.Linear(hidden, H))
        if kind == "mlp":
            w = (module[0].weight, module[0].bias, module[2].weight, module[2].bias)
        else:
            w = (module.weight, module.bias, None, None)
        wc = tuple(None if t is None else t.detach().to(dev, dtype).contiguous() for t in w)
        width = hd if kind == "mlp" else 0
        for S in (1, 4096, 32768, 131072):
            x = torch.randn(1, S, hidden, device=dev).to(dtype)
            k = torch.empty(1, H, S, 64, device=dev, dtype=dtype)
            iters = 200 if S <= 4096 else 50

            def ours():
                return native.kvzap_score(x, k, k, wc)

            def ref():
                m = module.to(dev, dtype=dtype).eval()
                with torch.no_grad():
                    return m(x).transpose(1, 2)

            t_ours, t_ref = timed(ours, iters), timed(ref, iters)
            # the same calls replayed from CUDA graphs: device time without the Python and launch overhead
            g_ours, g_ref = native.capture(ours), native.capture(ref)
            tg_ours, tg_ref = timed(g_ours.replay, iters), timed(g_ref.replay, iters)
            flop = 2 * S * hidden * width + 2 * S * max(width, 1) * H if width else 2 * S * hidden * H
            print(json.dumps({"case": f"{kind} score", "S": S, "ms": round(t_ours, 4), "ref_ms": round(t_ref, 4),
                              "graph_ms": round(tg_ours, 4), "ref_graph_ms": round(tg_ref, 4),
                              "tflops": round(flop / tg_ours / 1e9, 1), "ref_tflops": round(flop / tg_ref / 1e9, 1),
                              "card": name}), flush=True)
            del g_ours, g_ref
            module = module.float().cpu()
    S = 131072
    scores = torch.randn(1, H, S, device=dev).to(dtype)
    n_evict = S - 128
    t_ours = timed(lambda: native.threshold_evict(scores, n_evict, 0.0, 0), 50)
    t_ref = timed(lambda: torch.where(scores[..., :n_evict] < 0.0), 50)
    print(json.dumps({"case": "dms eviction", "S": S, "ms": round(t_ours, 4), "ref_ms": round(t_ref, 4),
                      "card": name}), flush=True)


if __name__ == "__main__":
    main()
