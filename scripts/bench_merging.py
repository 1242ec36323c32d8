"""Times the MergingPress kernels on the GPU and a torch restatement of the reference's merge beside them, in one run.

    python scripts/bench_merging.py [--sizes 4096,16384,32768,65536,131072] [--runs 3] [--json out.json]

At the Llama-3.1-8B layer shape (B 1, Hkv 8, D 128, bf16), Knorm scores, compression ratio 0.5, the reference defaults
(similarity_threshold 0, merge_fraction 1) and each sequence length S:
(a) `native.merging_compress` (selection, compaction and merge), replayed as a CUDA graph;
(b) `native.merging_merge` on the same kept positions (the merge alone), replayed as a CUDA graph;
(c) the reference's `MergingPress.merge` restated in torch (the dense fp32 [B, Hkv, n_evict, n_kept] similarity
    product, max, scatter_add_), only where its similarity tensor fits in device memory (S <= 32768 here).
Every shape is warmed up first; then they are timed in turn, `--runs` times over, each call between its own CUDA
events; every figure is the median over the runs of the per-run median. The useful work is the similarity product,
2 D n_evict n_kept FLOP per kv head; its rate is given as a share of the 989 TFLOP/s dense bf16 data-sheet figure of
the H100 SXM, which is not a measured peak. The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

DATASHEET_TFLOPS = 989.0
B, HKV, D = 1, 8, 128
REFERENCE_MAX_S = 32768


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


def reference_merge(keys, values, indices):
    """The reference's MergingPress.merge at its defaults, restated in torch: complement, gathers, normalised fp32 keys,
    the dense similarity product and its max, the weights, and scatter_add_ of the weighted evicted values."""
    b, h, s, d = keys.shape
    n_kept = indices.shape[2]
    mask = torch.ones(b, h, s, dtype=torch.bool, device=keys.device).scatter_(2, indices, False)
    ev = mask.nonzero()[:, 2].reshape(b, h, s - n_kept)
    ki, ei = indices.unsqueeze(-1).expand(-1, -1, -1, d), ev.unsqueeze(-1).expand(-1, -1, -1, d)
    kk, ke = keys.gather(2, ki).float(), keys.gather(2, ei).float()
    vk, ve = values.gather(2, ki), values.gather(2, ei)
    kk = kk / kk.norm(dim=-1, keepdim=True).clamp(min=1e-6)
    ke = ke / ke.norm(dim=-1, keepdim=True).clamp(min=1e-6)
    sim, target = (ke @ kk.transpose(-1, -2)).max(dim=-1)
    w = sim.clamp(min=0) * (sim >= 0).float()
    en, tn = ve.float().norm(dim=-1), vk.float().norm(dim=-1).gather(2, target)
    w = w * en / (en + tn + 1e-6)
    acc_v = torch.zeros(b, h, n_kept, d, device=keys.device).scatter_add_(
        2, target.unsqueeze(-1).expand(-1, -1, -1, d), w.unsqueeze(-1) * ve.float())
    acc_w = torch.zeros(b, h, n_kept, device=keys.device).scatter_add_(2, target, w)
    merged = torch.where((acc_w > 0).unsqueeze(-1), ((vk.float() + acc_v) / (1 + acc_w).unsqueeze(-1)).to(values.dtype),
                         vk)
    return values.clone().scatter_(2, ki, merged)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=str, default="4096,16384,32768,65536,131072")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_merging.py measures on a CUDA device; none is visible")
    from kvpress_b200 import native

    native.load()
    res = {"card": card(), "shape": {"B": B, "Hkv": HKV, "D": D, "dtype": "bf16", "scores": "knorm",
                                     "compression_ratio": 0.5, "similarity_threshold": 0.0, "merge_fraction": 1.0},
           "datasheet_tflops": DATASHEET_TFLOPS, "runs": args.runs,
           "note": "shares are against the H100 SXM dense bf16 data-sheet figure, not a measured peak"}
    sizes = [int(x) for x in args.sizes.split(",")]
    for S in sizes:
        g = torch.Generator(device="cuda").manual_seed(S)
        k = torch.randn((B, HKV, S, D), generator=g, device="cuda").to(torch.bfloat16)
        v = torch.randn((B, HKV, S, D), generator=g, device="cuda").to(torch.bfloat16)
        n_kept = S // 2
        scores = native.knorm_score(k)
        kept = native.scores_select(scores, n_kept)
        work = {
            "a": native.capture(lambda: native.merging_compress(scores, k, v, 0.0, 1.0, n_kept)).replay,
            "b": native.capture(lambda: native.merging_merge(k, v, kept, 0.0, 1.0)).replay,
        }
        if S <= REFERENCE_MAX_S:
            topk = scores.topk(n_kept, dim=-1).indices
            work["c"] = lambda: reference_merge(k, v, topk)
        reps = max(5, min(100, int(4e5 // S)))
        runs = {key: [] for key in work}
        for _ in range(args.runs):  # alternating
            for key in runs:
                runs[key].append(timed(work[key], reps if key != "c" else max(3, reps // 4)))
        med = {key: sorted(x)[len(x) // 2] for key, x in runs.items()}
        flop = 2.0 * D * (S - n_kept) * n_kept * B * HKV
        out = {"reps": reps, "similarity_flop": flop, "per_run_ms": {k_: [round(x, 4) for x in xs] for k_, xs in runs.items()}}
        for key, name in (("a", "a_compress"), ("b", "b_merge"), ("c", "c_reference_restated")):
            if key in med:
                tf = flop / (med[key] * 1e-3) / 1e12
                out[name] = {"median_ms": round(med[key], 4), "tflop_per_s": round(tf, 1),
                             "share_of_datasheet": round(tf / DATASHEET_TFLOPS, 3)}
        if "c" in med:
            out["c_over_b_speedup"] = round(med["c"] / med["b"], 2)
        else:
            out["c_reference_restated"] = f"not run: its similarity tensor takes {flop / D / 2 * 4 / 1e9:.1f} GB"
        res[f"S{S}"] = out
        print(json.dumps({f"S{S}": out, "card": res["card"]}), flush=True)
        del work
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(line + "\n")


if __name__ == "__main__":
    main()
