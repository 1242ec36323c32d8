"""Times the LagKV kernel on the GPU and the reference's score restated in torch beside it, in one run.

    python scripts/bench_lagkv.py [--sizes 4096,16384,32768,131072] [--runs 3] [--json out.json]

At the Llama-3.1-8B layer shape (B 1, Hkv 8, D 128, bf16), n_sink 4, lag_size 128 and each sequence length S:
(a) `native.lagkv_score` (ranks), replayed as a CUDA graph;
(b) `native.lagkv_compress` at compression ratio 0.5, replayed as a CUDA graph;
(c) the reference's `LagKVPress.score` restated in torch, in the cache dtype as the reference runs it.
Each is timed with CUDA events per call; every figure is the median over `--runs` runs of the per-run median. The
compulsory bytes are K and V read once (a, c), plus the kept rows of K and V read and written (b); the rates are given as
a share of the 3.35 TB/s data-sheet HBM3 bandwidth of the H100 SXM, which is not a measured peak. The card's name and
power limit are read in the same run.
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
B, HKV, D, N_SINK, LAG = 1, 8, 128, 4, 128


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


def reference_score(keys, values):
    """The reference's LagKVPress.score (kvpress/presses/lagkv_press.py), ranks, restated in torch."""
    bsz, heads, q_len, d = keys.shape
    end = N_SINK + ((q_len - N_SINK) // LAG) * LAG
    tail_len = LAG + q_len - end

    def states(target):
        ref, cur = target[:, :, 1:], target[:, :, :-1]
        min_r = ref.min(dim=-2).values.unsqueeze(-2).expand(-1, -1, -1, LAG, -1)
        max_r = ref.max(dim=-2).values.unsqueeze(-2).expand(-1, -1, -1, LAG, -1)
        return ((cur - min_r) / (max_r - min_r)).std(dim=-1).softmax(dim=-1)

    ks = states(keys[:, :, N_SINK:end].view(bsz, heads, -1, LAG, d))
    vs = states(values[:, :, N_SINK:end].view(bsz, heads, -1, LAG, d))
    score = ((ks + vs) / 2).argsort(dim=-1).argsort(dim=-1) / LAG
    score = score.to(keys.dtype)
    sink = torch.ones((bsz, heads, N_SINK), dtype=score.dtype, device=score.device)
    tail = torch.ones((bsz, heads, tail_len), dtype=score.dtype, device=score.device)
    return torch.cat((sink, score.reshape(bsz, heads, -1), tail), dim=-1)


def rates(ms: float, nbytes: float) -> dict:
    tbps = nbytes / (ms * 1e-3) / 1e12
    return {"median_ms": round(ms, 4), "compulsory_tb_per_s": round(tbps, 2),
            "share_of_datasheet_bw": round(tbps / DATASHEET_TBPS, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=str, default="4096,16384,32768,131072")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_lagkv.py measures on a CUDA device; none is visible")
    from kvpress_b200 import native

    native.load()
    res = {"card": card(), "shape": {"B": B, "Hkv": HKV, "D": D, "dtype": "bf16", "n_sink": N_SINK, "lag_size": LAG},
           "datasheet_tb_per_s": DATASHEET_TBPS, "runs": args.runs,
           "note": "shares are against the H100 SXM data-sheet bandwidth, not a measured peak"}
    for S in (int(x) for x in args.sizes.split(",")):
        reps = max(10, min(200, int(8e6 // S)))
        g = torch.Generator(device="cuda").manual_seed(S)
        k = torch.randn((B, HKV, S, D), generator=g, device="cuda").to(torch.bfloat16)
        v = torch.randn((B, HKV, S, D), generator=g, device="cuda").to(torch.bfloat16)
        n_kept = S // 2
        kv_bytes = 2.0 * 2 * B * HKV * S * D
        kept_bytes = 2.0 * 2 * 2 * B * HKV * n_kept * D
        ga = native.capture(lambda: native.lagkv_score(k, v, N_SINK, LAG, False))
        gb = native.capture(lambda: native.lagkv_compress(k, v, N_SINK, LAG, False, n_kept))
        runs = {"a": [], "b": [], "c": []}
        for _ in range(args.runs):
            runs["a"].append(timed(ga.replay, reps))
            runs["b"].append(timed(gb.replay, reps))
            runs["c"].append(timed(lambda: reference_score(k, v), max(5, reps // 4)))
        med = {key: sorted(x)[len(x) // 2] for key, x in runs.items()}
        out = {"reps": reps, "kv_bytes": kv_bytes, "kept_rows_bytes": kept_bytes,
               "a_score": rates(med["a"], kv_bytes), "b_compress_r0.5": rates(med["b"], kv_bytes + kept_bytes),
               "c_reference_restated": rates(med["c"], kv_bytes),
               "per_run_ms": {key: [round(x, 4) for x in xs] for key, xs in runs.items()}}
        out["a_over_c_speedup"] = round(med["c"] / med["a"], 2)
        del ga, gb, k, v
        torch.cuda.empty_cache()
        res[f"S{S}"] = out
        print(json.dumps({f"S{S}": out}), flush=True)
    line = json.dumps(res)
    print(line)
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(line + "\n")


if __name__ == "__main__":
    main()
