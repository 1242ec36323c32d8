"""Times the CriticalKV score kernel on the GPU and the reference's per-head path beside it, in one run.

    python scripts/bench_criticalkv.py [--reps 20] [--json out.json]

(a) `native.criticalkv_score` at the Llama-3.1-8B layer shape at 128k (Hq 32, Hkv 8, D 128, hidden 4096) and at the
    Llama-3.1-70B shape at 32k (Hq 64, Hkv 8, hidden 8192);
(b) the full CriticalKVPress(ExpectedAttentionPress(use_vnorm=False)) sequence at the 8B 128k shape: the EA score,
    then the CriticalKV compress at compression ratio 0.5;
(c) a torch restatement of the reference's vwl1norm (kvpress/presses/criticalkv_press.py:57-76): per query head a
    [S, D] x [D, hidden] matmul in the cache dtype, its L1 norm over hidden, the mean over the group.
(a) and (b) are replayed as CUDA graphs, (c) runs eagerly (it allocates); all are timed with CUDA events. Rates are
computed from shape FLOPs (2 Hq S D hidden) and compared with the 989 TFLOP/s dense BF16 data-sheet figure of the H100
SXM, which is not a measured peak. At the timed size the kernel's norms are checked against an fp32 torch evaluation on
sampled positions of every row.
"""
from __future__ import annotations

import argparse
import json
import math
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

DATASHEET_TFLOPS = 989.0
SHAPES = {  # name -> (B, Hkv, Hq, S, D, hidden)
    "llama8b_128k": (1, 8, 32, 131072, 128, 4096),
    "llama70b_32k": (1, 8, 64, 32768, 128, 8192),
}


def card() -> dict:
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        out["power_limit"], out["max_sm_clock"] = [x.strip() for x in q.split(",")]
    except Exception as e:  # noqa: BLE001 — reported, not hidden
        out["power_limit"] = f"unavailable ({e})"
    return out


def timed(fn, reps: int) -> list:
    """Per-call milliseconds of `reps` calls, each between its own CUDA events, after two warm-up calls."""
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return sorted(a.elapsed_time(b) for a, b in ev)


def summary(ms: list, flops: float) -> dict:
    med = ms[len(ms) // 2]
    tflops = flops / (med * 1e-3) / 1e12
    return {"median_ms": round(med, 4), "min_ms": round(ms[0], 4), "max_ms": round(ms[-1], 4),
            "tflops": round(tflops, 1), "share_of_datasheet": round(tflops / DATASHEET_TFLOPS, 3)}


def inputs(shape, dtype=torch.bfloat16, seed=0):
    B, Hkv, Hq, S, D, hidden = shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    v = torch.randn((B, Hkv, S, D), generator=g, device="cuda", dtype=torch.float32).to(dtype)
    wo = (torch.randn((hidden, Hq * D), generator=g, device="cuda", dtype=torch.float32) / math.sqrt(Hq * D)).to(dtype)
    base = torch.rand((B, Hkv, S), generator=g, device="cuda", dtype=torch.float32).to(dtype)
    return v, wo, base


def reference_vwl1norm(values, wo, Hq):
    """criticalkv_press.py:58-76 restated: Wo^T viewed [Hq, D, hidden], per head V_h @ Wo_h, L1 over hidden."""
    B, Hkv, S, D = values.shape
    G = Hq // Hkv
    w = wo.transpose(0, 1).view(Hq, D, wo.shape[0])
    norms = [torch.norm(values[:, h // G].matmul(w[h].unsqueeze(0)), p=1, dim=-1) for h in range(Hq)]
    return torch.stack(norms, dim=1).view(B, Hkv, G, S).mean(dim=2)


def check_norms(native, v, wo, Hq, n_sample=512) -> dict:
    """Kernel norms (base = 0, epsilon = 1: score = norm rounded once) against fp32 torch on sampled positions."""
    B, Hkv, S, D = v.shape
    G = Hq // Hkv
    got = native.criticalkv_score(torch.zeros(v.shape[:3], dtype=v.dtype, device=v.device), v, wo, 1.0, 0)
    pos = torch.randperm(S, device=v.device)[:n_sample].sort().values
    w = wo.float()
    ref = torch.zeros((B, Hkv, pos.numel()), device=v.device)
    for h in range(Hq):
        ref[:, h // G] += (v[:, h // G, pos].float() @ w[:, h * D:(h + 1) * D].T).abs().sum(-1)
    ref /= G
    rel = ((got[..., pos].float() - ref) / ref).abs().max().item()
    return {"max_rel_err": rel, "bound": 2.0 ** -8, "ok": rel <= 2.0 ** -8}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_criticalkv.py measures on a CUDA device; none is visible")
    from kvpress_b200 import native

    native.load()
    res = {"card": card(), "datasheet_tflops_bf16_dense": DATASHEET_TFLOPS,
           "note": "share_of_datasheet is against the H100 SXM data-sheet figure, not a measured peak"}
    for name, shape in SHAPES.items():
        B, Hkv, Hq, S, D, hidden = shape
        v, wo, base = inputs(shape)
        flops = 2.0 * B * Hq * S * D * hidden
        g = native.capture(lambda: native.criticalkv_score(base, v, wo, 1e-4, S // 4))
        res[f"a_score_{name}"] = summary(timed(g.replay, args.reps), flops)
        res[f"a_score_{name}"]["norm_check"] = check_norms(native, v, wo, Hq)
        del g
        if name == "llama8b_128k":
            k = torch.randn_like(v)
            mu = torch.randn((B, Hq, D), device="cuda").to(v.dtype) * 0.1
            cov = (torch.randn((B, Hq, D, D), device="cuda") * 0.01).to(v.dtype)
            ratio = 0.5
            n_kept = int(S * (1 - ratio))
            n_first = int((1 - ratio) * S * 0.5)

            def press_sequence():
                sc = native.expected_attention_score(k, v, mu, cov, 0.0, 4, False)
                return native.criticalkv_compress(sc, k, v, wo, 1e-4, n_first, n_kept)

            g = native.capture(press_sequence)
            res[f"b_press_{name}"] = summary(timed(g.replay, args.reps), flops)
            del g
            torch.cuda.empty_cache()
            got = reference_vwl1norm(v, wo, Hq)  # warm-up and a sanity check of the restatement
            kern = native.criticalkv_score(torch.zeros_like(base), v, wo, 1.0, 0).float()
            res[f"c_reference_{name}"] = summary(timed(lambda: reference_vwl1norm(v, wo, Hq), max(3, args.reps // 4)),
                                                 flops)
            res[f"c_reference_{name}"]["max_rel_diff_to_kernel"] = float(((got.float() - kern) / kern).abs().max())
            del got, kern
            torch.cuda.empty_cache()
        del v, wo, base
        torch.cuda.empty_cache()
    a, c = res["a_score_llama8b_128k"]["median_ms"], res["c_reference_llama8b_128k"]["median_ms"]
    res["a_over_c_speedup_llama8b_128k"] = round(c / a, 2)
    line = json.dumps(res)
    print(line)
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(line + "\n")


if __name__ == "__main__":
    main()
