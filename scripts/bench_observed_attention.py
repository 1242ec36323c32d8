"""Times the ObservedAttention (H2O) kernels on the GPU and the reference's eager-attention path beside them, in one run.

    python scripts/bench_observed_attention.py [--sizes 4096,16384,32768,131072] [--json out.json]

At the Llama-3.1-8B layer shape (B 1, Hkv 8, Hq 32, D 128, bf16) and each sequence length S (n_q = S, prefill):
(a) `native.observed_attention_score`, replayed as a CUDA graph;
(b) `native.observed_attention_compress` at compression ratio 0.5, replayed as a CUDA graph;
(c) (a) with the torch prologue of the press: q_proj over the S hidden states, then RoPE;
(d) where it fits, the reference's layer path restated in torch as eager attention does it: repeat_kv, q k^T * scaling
    in bf16, the causal mask, the fp32 softmax cast to bf16, then the press's sum over the queries, the division by
    arange(S, 0, -1) in bf16 and the mean over the group.
All are timed with CUDA events, per call. Rates count two passes of 2 D Hq n_q (n_q + 1) / 2 FLOP (70.4 TFLOP per pass
at 128k) and are compared with the 989 TFLOP/s dense BF16 data-sheet figure of the H100 SXM, which is not a measured
peak. Each pass also needs Hq n_q (n_q + 1) / 2 exponentials (2.75e11 at 128k). The card's name and power limit are read
in the same run. Where (d) runs, the kernel's scores are compared with it.
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
B, HKV, HQ, D, HIDDEN = 1, 8, 32, 128, 4096
# the eager restatement holds [Hq, S, S] in bf16, then twice in fp32 (softmax's cast input and its output): 80 GiB at
# 16k, which an 80 GB card does not hold; the attempt is reported
REFERENCE_MAX_S = 16384


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


def flops(S: int) -> float:
    """Two passes (row statistics, column sums) of the causal q k^T: 2 D Hq n_q (n_q + 1) / 2 each, n_q = S."""
    return 2 * (2.0 * D * HQ * S * (S + 1) / 2)


def summary(ms: list, S: int) -> dict:
    med = ms[len(ms) // 2]
    tflops = flops(S) / (med * 1e-3) / 1e12
    return {"median_ms": round(med, 4), "min_ms": round(ms[0], 4), "max_ms": round(ms[-1], 4),
            "tflops": round(tflops, 1), "share_of_datasheet": round(tflops / DATASHEET_TFLOPS, 3)}


def rope(S: int):
    inv_freq = 1.0 / (500000.0 ** (torch.arange(0, D, 2, device="cuda").float() / D))
    ang = torch.arange(S, device="cuda").float()[:, None] * inv_freq[None]
    emb = torch.cat([ang, ang], dim=-1)[None]
    return emb.cos().to(torch.bfloat16), emb.sin().to(torch.bfloat16)


def reference_layer(q, k, scaling):
    """The reference's path on one layer: eager attention's weights, then ObservedAttentionPress.score."""
    S = k.shape[2]
    G = HQ // HKV
    kr = k[:, :, None].expand(B, HKV, G, S, D).reshape(B, HQ, S, D)
    w = torch.matmul(q, kr.transpose(2, 3)).mul_(scaling)  # in place: the same bf16 values, one [Hq, S, S] less
    w.masked_fill_(torch.ones((S, S), dtype=torch.bool, device="cuda").triu_(1), float("-inf"))
    p = torch.softmax(w, dim=-1, dtype=torch.float32)
    del w
    p16 = p.to(q.dtype)
    del p
    scores = p16.sum(2) / torch.arange(S, 0, -1, device="cuda").to(q.dtype)
    del p16
    return scores.view(B, HKV, G, S).mean(2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=str, default="4096,16384,32768,131072")
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_observed_attention.py measures on a CUDA device; none is visible")
    from kvpress_b200 import native
    from kvpress_b200.utils import apply_rope

    native.load()
    res = {"card": card(), "shape": {"B": B, "Hkv": HKV, "Hq": HQ, "D": D, "dtype": "bf16", "n_q": "S"},
           "datasheet_tflops_bf16_dense": DATASHEET_TFLOPS,
           "note": "share_of_datasheet is against the H100 SXM data-sheet figure, not a measured peak"}
    scaling = D ** -0.5
    for S in (int(x) for x in args.sizes.split(",")):
        reps = max(3, min(50, int(4e5 // S)))
        g = torch.Generator(device="cuda").manual_seed(S)
        k = torch.randn((B, HKV, S, D), generator=g, device="cuda").to(torch.bfloat16)
        v = torch.randn((B, HKV, S, D), generator=g, device="cuda").to(torch.bfloat16)
        q = (1.5 * torch.randn((B, HQ, S, D), generator=g, device="cuda")).to(torch.bfloat16)
        out = {"flop_per_call": flops(S), "exp2_per_call": 2.0 * HQ * S * (S + 1) / 2, "reps": reps}
        ga = native.capture(lambda: native.observed_attention_score(k, q, scaling))
        out["a_score"] = summary(timed(ga.replay, reps), S)
        gb = native.capture(lambda: native.observed_attention_compress(k, v, q, scaling, S // 2))
        out["b_compress_r0.5"] = summary(timed(gb.replay, reps), S)
        del gb
        hidden = (torch.randn((B, S, HIDDEN), generator=g, device="cuda") * 0.5).to(torch.bfloat16)
        q_proj = (torch.randn((HQ * D, HIDDEN), generator=g, device="cuda") / math.sqrt(HIDDEN)).to(torch.bfloat16)
        cos, sin = rope(S)

        def with_prologue():
            qq = torch.nn.functional.linear(hidden, q_proj).view(B, S, HQ, D).transpose(1, 2)
            return native.observed_attention_score(k, apply_rope(qq, cos, sin).contiguous(), scaling)

        out["c_score_with_prologue"] = summary(timed(with_prologue, reps), S)
        del hidden, q_proj, cos, sin
        torch.cuda.empty_cache()
        if S <= REFERENCE_MAX_S:
            try:
                ref = reference_layer(q, k, scaling).float()
                kern = ga.replay().float()
                torch.cuda.synchronize()
                out["d_reference_eager"] = summary(timed(lambda: reference_layer(q, k, scaling), max(3, reps // 4)), S)
                out["d_reference_eager"]["max_rel_diff_to_kernel"] = float(((kern - ref).abs() / ref.abs()).max())
                out["a_over_d_speedup"] = round(out["d_reference_eager"]["median_ms"] / out["a_score"]["median_ms"], 2)
                del ref, kern
            except torch.OutOfMemoryError as e:
                out["d_reference_eager"] = f"out of memory ({str(e).splitlines()[0]})"
        else:
            out["d_reference_eager"] = "not run: [Hq, S, S] weights exceed the card's memory"
        del ga, k, v, q
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
