"""Times the ThinK prune on the GPU and the reference's compress body restated in torch beside it, in one run.

    python scripts/bench_think.py [--sizes 4096,32768,131072] [--runs 3] [--json out.json]

At the Llama-3.1-8B layer shape (B 1, Hkv 8, Hq 32, D 128, bf16), window 32 and key_channel_compression_ratio 0.5
(64 channels pruned), for each sequence length S:
(a) `native.think_prune` on one K buffer, replayed as a CUDA graph. Repeated prunes of one buffer do the same work: the
    kernels' reads and writes do not depend on the values (the zero pass rewrites every 16-byte vector that holds a
    pruned channel, whether it is already zero or not);
(b) the reference's compress body restated in torch (pow, mean, view-mean, product, topk, scatter_), in the cache dtype
    as the reference runs it;
(c) at 32k only, `ComposedPress([SnapKVPress(0.5), ThinKPress(0.5)])`'s two native calls (SnapKV compress, then the
    prune of its kept keys), for context.
Each is timed with CUDA events per call; every figure is the median over `--runs` runs of the per-run median. The
compulsory bytes of (a) are K read once plus the pruned half of K written; the share is against the 3.35 TB/s
data-sheet HBM3 bandwidth of the H100 SXM, which is not a measured peak. The card's name and power limit are read in
the same run.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

DATASHEET_TBPS = 3.35
B, HKV, HQ, D, W, RATIO = 1, 8, 32, 128, 32, 0.5


def card() -> dict:
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        out["power_limit"], out["max_sm_clock"] = [x.strip() for x in q.split(",")]
    except Exception as e:  # noqa: BLE001 — reported, not hidden
        out["power_limit"] = f"unavailable ({e})"
    return out


def timed(fn, reps: int) -> float:
    """Median milliseconds of `reps` calls, each between its own CUDA events, after two warm-up calls."""
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    ms = sorted(a.elapsed_time(b) for a, b in ev)
    return ms[len(ms) // 2]


def reference_prune(keys, queries, n_pruned):
    """The reference's ThinKPress.compress body (kvpress/presses/think_press.py) restated in torch."""
    bsz, num_key_value_heads, k_len, head_dim = keys.shape
    queries_norm = torch.pow(queries, 2).mean(dim=2)
    queries_norm = queries_norm.view(bsz, num_key_value_heads, HQ // num_key_value_heads, head_dim).mean(2)
    keys_norm = torch.pow(keys, 2).mean(dim=2)
    key_scores = queries_norm * keys_norm
    indices = key_scores.topk(n_pruned, dim=-1, largest=False).indices
    indices = indices.unsqueeze(2).expand(-1, -1, k_len, -1)
    return keys.scatter_(-1, indices, 0)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="4096,32768,131072")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_think.py measures on the GPU and has no CPU fallback")
    from kvpress_b200 import native

    native.load()
    dev = torch.device("cuda:0")
    n_pruned = int(D * RATIO)
    result = {"card": card(), "shape": dict(B=B, Hkv=HKV, Hq=HQ, D=D, window=W, n_pruned=n_pruned), "sizes": {}}
    g = torch.Generator(device=dev).manual_seed(0)
    for S in (int(s) for s in args.sizes.split(",")):
        k = torch.randn(B, HKV, S, D, generator=g, device=dev).to(torch.bfloat16)
        q = torch.randn(B, HQ, W, D, generator=g, device=dev).to(torch.bfloat16)
        graph = native.capture(lambda: native.think_prune(k, q, n_pruned))
        kern = [timed(graph.replay, args.reps) for _ in range(args.runs)]
        torch_ms = [timed(lambda: reference_prune(k, q, n_pruned), args.reps) for _ in range(args.runs)]
        ms = sorted(kern)[len(kern) // 2]
        ref_ms = sorted(torch_ms)[len(torch_ms) // 2]
        bytes_ = B * HKV * S * D * 2 + B * HKV * S * n_pruned * 2
        row = {"think_prune_ms": ms, "torch_reference_ms": ref_ms, "compulsory_bytes": bytes_,
               "share_of_datasheet_bw": bytes_ / (ms * 1e-3) / (DATASHEET_TBPS * 1e12)}
        if S == 32768:
            v = torch.randn_like(k)
            qs = torch.randn(B, HQ, 64, D, generator=g, device=dev).to(torch.bfloat16)

            def composed():
                k_out, _, _, _ = native.snapkv_compress(k, v, qs, 64, 5, S // 2)
                native.think_prune(k_out, q, n_pruned)

            row["snapkv_then_think_ms"] = sorted(timed(composed, args.reps) for _ in range(args.runs))[args.runs // 2]
        result["sizes"][S] = row
        print(S, json.dumps(row), flush=True)
        del graph
    print(json.dumps(result))
    if args.json:
        Path(args.json).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
