"""Times the NonCausalAttention kernel on the GPU and the reference's layer path beside it, in one run.

    python scripts/bench_non_causal_attention.py [--sizes 4096,16384,32768,131072] [--json out.json]

At the Llama-3.1-8B layer shape (B 1, Hkv 8, Hq 32, D 128, bf16, chunk_size 256) and each sequence length S:
(a) `native.non_causal_attention_score`, replayed as a CUDA graph;
(b) `native.non_causal_attention_compress` at compression ratio 0.5, replayed as a CUDA graph;
(c) (a) with the torch prologue of the press: q_proj over the S hidden states, then RoPE;
(d) the reference's layer path restated in torch: repeat_kv, the [B, Hq, S/cs, cs, cs] logits in bf16, the padding
    masks, the fp32 softmax, the sum over the queries, the group mean, ||v||, the pooling and the z-score.
All are timed with CUDA events, per call. The kernel needs 2 x 2 D Hq S cs FLOP (pass A and the recomputed pass B: 5.5e11
at 128k), 2 Hq S cs exponentials and reads Q (1 GiB at 128k), K and V once. Rates are compared with the 989 TFLOP/s
dense BF16 and 3.35 TB/s data-sheet figures of the H100 SXM, which are not measured peaks. The card's name and power
limit are read in the same run; the overlap of the kernel's and the restatement's selections at r = 0.5 is reported.
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

DATASHEET_TFLOPS = 989.0
DATASHEET_TBPS = 3.35
B, HKV, HQ, D, HIDDEN, CS = 1, 8, 32, 128, 4096, 256


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
    """Pass A and pass B of the kernel: 2 D Hq S cs each (the padded last chunk counted whole)."""
    return 2 * (2.0 * D * HQ * (-(-S // CS) * CS) * CS)


def compulsory_bytes(S: int) -> float:
    return 2.0 * S * D * (HQ + 2 * HKV)


def summary(ms: list, S: int) -> dict:
    med = ms[len(ms) // 2]
    tflops = flops(S) / (med * 1e-3) / 1e12
    tbps = compulsory_bytes(S) / (med * 1e-3) / 1e12
    return {"median_ms": round(med, 4), "min_ms": round(ms[0], 4), "max_ms": round(ms[-1], 4),
            "tflops": round(tflops, 1), "share_of_datasheet_flops": round(tflops / DATASHEET_TFLOPS, 3),
            "compulsory_tb_per_s": round(tbps, 2), "share_of_datasheet_bw": round(tbps / DATASHEET_TBPS, 3)}


def rope(S: int):
    inv_freq = 1.0 / (500000.0 ** (torch.arange(0, D, 2, device="cuda").float() / D))
    ang = torch.arange(S, device="cuda").float()[:, None] * inv_freq[None]
    emb = torch.cat([ang, ang], dim=-1)[None]
    return emb.cos().to(torch.bfloat16), emb.sin().to(torch.bfloat16)


def reference_layer(q, k, v):
    """The reference's NonCausalAttnPress.score on one layer, from the RoPE'd queries."""
    S = k.shape[2]
    G = HQ // HKV
    kr = k[:, :, None].expand(B, HKV, G, S, D).reshape(B, HQ, S, D)
    n = -(-S // CS)
    pad = n * CS - S
    qp = F.pad(q, (0, 0, 0, pad)).view(B, HQ, n, CS, D)
    kp = F.pad(kr, (0, 0, 0, pad)).view(B, HQ, n, CS, D)
    dots = torch.matmul(qp, kp.transpose(-2, -1))
    if pad:
        dots[:, :, -1, CS - pad:, :] = 0
        dots[:, :, -1, :, CS - pad:] = -1e-9
    attn = torch.softmax(dots.to(torch.float32), dim=-1)
    del dots
    A = attn.sum(dim=-2).view(B, HQ, n * CS)[..., :S]
    del attn
    A = A.view(B, HKV, G, S).mean(dim=2)
    x = F.avg_pool1d(A * v.norm(dim=-1), kernel_size=3, padding=1, stride=1)
    return (x - x.mean()) / x.std().clamp_min(1e-6)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=str, default="4096,16384,32768,131072")
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_non_causal_attention.py measures on a CUDA device; none is visible")
    from kvpress_b200 import native
    from kvpress_b200.utils import apply_rope

    native.load()
    res = {"card": card(), "shape": {"B": B, "Hkv": HKV, "Hq": HQ, "D": D, "dtype": "bf16", "chunk_size": CS},
           "datasheet_tflops_bf16_dense": DATASHEET_TFLOPS, "datasheet_tb_per_s": DATASHEET_TBPS,
           "note": "shares are against the H100 SXM data-sheet figures, not measured peaks"}
    for S in (int(x) for x in args.sizes.split(",")):
        reps = max(5, min(50, int(2e6 // S)))
        g = torch.Generator(device="cuda").manual_seed(S)
        sig = 8 ** 0.5 / D ** 0.25  # unscaled logits of standard deviation about 8
        k = (sig * torch.randn((B, HKV, S, D), generator=g, device="cuda")).to(torch.bfloat16)
        v = torch.randn((B, HKV, S, D), generator=g, device="cuda").to(torch.bfloat16)
        q = (sig * torch.randn((B, HQ, S, D), generator=g, device="cuda")).to(torch.bfloat16)
        out = {"flop_per_call": flops(S), "exp2_per_call": 2.0 * HQ * (-(-S // CS) * CS) * CS,
               "compulsory_bytes": compulsory_bytes(S), "reps": reps}
        ga = native.capture(lambda: native.non_causal_attention_score(k, v, q, CS))
        out["a_score"] = summary(timed(ga.replay, reps), S)
        gb = native.capture(lambda: native.non_causal_attention_compress(k, v, q, CS, S // 2, return_indices=True))
        out["b_compress_r0.5"] = summary(timed(gb.replay, reps), S)
        idx_kernel = gb.replay()[2].long()
        hidden = (torch.randn((B, S, HIDDEN), generator=g, device="cuda") * 0.5).to(torch.bfloat16)
        q_proj = (torch.randn((HQ * D, HIDDEN), generator=g, device="cuda") / math.sqrt(HIDDEN)).to(torch.bfloat16)
        cos, sin = rope(S)

        def with_prologue():
            qq = torch.nn.functional.linear(hidden, q_proj).view(B, S, HQ, D).transpose(1, 2)
            return native.non_causal_attention_score(k, v, apply_rope(qq, cos, sin).contiguous(), CS)

        out["c_score_with_prologue"] = summary(timed(with_prologue, reps), S)
        del hidden, q_proj, cos, sin, gb
        torch.cuda.empty_cache()
        try:
            ref = reference_layer(q, k, v)
            idx_ref = ref.topk(S // 2, dim=-1).indices
            kept = torch.zeros((B, HKV, S), dtype=torch.bool, device="cuda")
            kept.scatter_(-1, idx_ref, True)
            out["selection_overlap"] = round(float(kept.gather(-1, idx_kernel).float().mean()), 4)
            del ref, kept, idx_ref
            torch.cuda.empty_cache()
            out["d_reference_restated"] = summary(timed(lambda: reference_layer(q, k, v), max(3, reps // 4)), S)
            out["a_over_d_speedup"] = round(out["d_reference_restated"]["median_ms"] / out["a_score"]["median_ms"], 2)
        except torch.OutOfMemoryError as e:
            out["d_reference_restated"] = f"out of memory ({str(e).splitlines()[0]})"
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
