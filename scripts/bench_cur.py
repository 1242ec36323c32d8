"""Times the CUR kernels on the GPU and the reference's score restated in torch beside them, in one run.

    python scripts/bench_cur.py [--sizes 4096,32768,131072] [--runs 3] [--json out.json]

At the Llama-3.1-8B layer shape (B 1, Hkv 8, D 128, bf16), the reference defaults (num_sinks 4, kv_product, windows of 16)
and each sequence length S:
(a) `native.cur_score`, replayed as a CUDA graph;
(b) `native.cur_compress` at compression ratio 0.5, replayed as a CUDA graph;
(c) the reference's `CURPress.score` restated in torch, in the cache dtype as the reference runs it;
(d) `native.cur_score` with a projection G [128, 20], replayed as a CUDA graph (the reference raises on a 16-bit cache
    here, so it has no counterpart).
Every shape is warmed up first; then the four are timed in turn, `--runs` times over, each call between its own CUDA
events; every figure is the median over the runs of the per-run median. The compulsory bytes are K and V read once and
the scores written (a, c, d), plus the kept rows of K and V read and written (b); the rates are given as a share of the
3.35 TB/s data-sheet HBM3 bandwidth of the H100 SXM, which is not a measured peak. The card's name and power limit are
read in the same run.
"""
from __future__ import annotations

import argparse
import json
import math
import subprocess
import sys
from pathlib import Path

import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

DATASHEET_TBPS = 3.35
B, HKV, D, SINKS, WINDOW, RANK = 1, 8, 128, 4, 16, 20


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
    """The reference's CURPress.score (kvpress/presses/cur_press.py) at its defaults, restated in torch."""
    k2 = (keys ** 2).sum(dim=-1)
    v2 = (values ** 2).sum(dim=-1)
    b, h, n = k2.shape
    pad = (WINDOW - n % WINDOW) % WINDOW
    k2 = F.pad(k2, (0, pad)).reshape(b, h, -1, WINDOW)
    k2 = (k2 / k2.sum(dim=-1, keepdim=True)).reshape(b, h, -1)[:, :, :n]
    v2 = F.pad(v2, (0, pad)).reshape(b, h, -1, WINDOW)
    v2 = (v2 / v2.sum(dim=-1, keepdim=True)).reshape(b, h, -1)[:, :, :n]
    scores = k2 * v2
    scores /= scores.sum(dim=-1, keepdim=True)
    scores[:, :, :SINKS] = 1.0
    return scores


def rates(ms: float, nbytes: float) -> dict:
    tbps = nbytes / (ms * 1e-3) / 1e12
    return {"median_ms": round(ms, 4), "compulsory_tb_per_s": round(tbps, 3),
            "share_of_datasheet_bw": round(tbps / DATASHEET_TBPS, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=str, default="4096,32768,131072")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_cur.py measures on a CUDA device; none is visible")
    from kvpress_b200 import native

    native.load()
    res = {"card": card(), "shape": {"B": B, "Hkv": HKV, "D": D, "dtype": "bf16", "num_sinks": SINKS,
                                     "leverage_type": "kv_product", "local_window_size": WINDOW, "r": RANK},
           "datasheet_tb_per_s": DATASHEET_TBPS, "runs": args.runs,
           "note": "shares are against the H100 SXM data-sheet bandwidth, not a measured peak"}
    sizes = [int(x) for x in args.sizes.split(",")]
    work = {}
    for S in sizes:  # every shape is captured (and so warmed up) before anything is timed
        g = torch.Generator(device="cuda").manual_seed(S)
        k = torch.randn((B, HKV, S, D), generator=g, device="cuda").to(torch.bfloat16)
        v = torch.randn((B, HKV, S, D), generator=g, device="cuda").to(torch.bfloat16)
        G = torch.randn((D, RANK), generator=g, device="cuda") / math.sqrt(RANK)
        work[S] = {
            "k": k, "v": v,
            "a": native.capture(lambda k=k, v=v: native.cur_score(k, v, SINKS, "kv_product", WINDOW)).replay,
            "b": native.capture(lambda k=k, v=v, n=S // 2: native.cur_compress(k, v, SINKS, "kv_product", WINDOW, None,
                                                                                n)).replay,
            "c": lambda k=k, v=v: reference_score(k, v),
            "d": native.capture(lambda k=k, v=v, G=G: native.cur_score(k, v, SINKS, "kv_product", WINDOW, G)).replay,
        }
        reference_score(k, v)
    torch.cuda.synchronize()
    for S in sizes:
        reps = max(10, min(200, int(8e6 // S)))
        n_kept = S // 2
        score_bytes = 2.0 * 2 * B * HKV * S * D + 2.0 * B * HKV * S
        kept_bytes = 2.0 * 2 * 2 * B * HKV * n_kept * D
        runs = {"a": [], "b": [], "c": [], "d": []}
        for _ in range(args.runs):  # alternating
            for key in runs:
                runs[key].append(timed(work[S][key], reps if key != "c" else max(5, reps // 4)))
        med = {key: sorted(x)[len(x) // 2] for key, x in runs.items()}
        out = {"reps": reps, "score_bytes": score_bytes, "kept_rows_bytes": kept_bytes,
               "a_score": rates(med["a"], score_bytes), "b_compress_r0.5": rates(med["b"], score_bytes + kept_bytes),
               "c_reference_restated": rates(med["c"], score_bytes), "d_score_projected_r20": rates(med["d"], score_bytes),
               "per_run_ms": {key: [round(x, 4) for x in xs] for key, xs in runs.items()}}
        out["a_over_c_speedup"] = round(med["c"] / med["a"], 2)
        res[f"S{S}"] = out
        print(json.dumps({f"S{S}": out, "card": res["card"]}), flush=True)
    line = json.dumps(res)
    print(line)
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(line + "\n")


if __name__ == "__main__":
    main()
