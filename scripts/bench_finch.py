"""Times FinchPress's score and compress on the GPU, and the reference's score + compress restated in torch beside them.

    python scripts/bench_finch.py [--sizes 4096,32768,131072] [--windows 64,512,2048] [--reps 10] [--json out.json]

At the Llama-3.1-8B layer shape (B 1, Hkv 8, Hq 32, D 128, bf16), compression_ratio 0.5 and rerotate_keys on, for each
sequence length S and window w (the question's length):
(a) `native.finch_score`;
(b) `native.finch_compress` unchunked and with chunk_length 4096, keys re-rotated; at w = 64 also with chunk_length S
    (one chunk per row: one CTA per row finds its threshold) and 5 (about S / 5 chunk CTAs per row);
(c) the reference's FinchPress.score + compress body restated in torch (repeat_kv, [B, Hq, w, S] logits, mask, fp32
    softmax, weighted means, topk, sort, re-rotation and gathers), unchunked; "oom" where it does not fit.
Each is the median of `--reps` calls between CUDA events after two warm-up calls. The achieved rate is
4 B Hq w S D flops (the two passes' QK^T products) over (a)'s time, beside the 989 TFLOP/s dense BF16 data-sheet figure
of the H100 SXM, which is not a measured peak. The card's name and power limit are read in the same run.
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

DATASHEET_TFLOPS = 989
B, HKV, HQ, D, RATIO, CHUNK = 1, 8, 32, 128, 0.5, 4096


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


def reference(k, v, q, w, inv_freq):
    """FinchPress.score + compress of the reference, restated in torch (unchunked, rerotate_keys)."""
    S = k.shape[2]
    G = HQ // HKV
    kr = k.repeat_interleave(G, dim=1)
    logits = torch.matmul(q, kr.transpose(2, 3)) / math.sqrt(D)
    mask = torch.ones_like(logits[0, 0], dtype=torch.bool).triu(S - w + 1)
    logits = logits.masked_fill(mask, float("-inf"))
    attn = torch.softmax(logits, dim=-1, dtype=torch.float32).to(q.dtype)[..., : S - w]
    del logits
    attn = attn * torch.arange(S - w, S, device=k.device)[None, None, :, None]
    scores = attn.mean(dim=-2).view(B, HKV, G, S - w).mean(dim=2)
    scores = torch.nn.functional.pad(scores, (0, w), value=scores.max().item() + 1)
    idx = scores.topk(int(S * (1 - RATIO)), dim=-1).indices.sort(dim=-1).values
    delta = (torch.arange(idx.shape[-1], device=k.device) - idx).float()[..., None] * inv_freq
    cos, sin = torch.cat((delta.cos(),) * 2, -1).to(k.dtype), torch.cat((delta.sin(),) * 2, -1).to(k.dtype)
    g = idx[..., None].expand(-1, -1, -1, D)
    kk = k.gather(2, g)
    rot = torch.cat((-kk[..., D // 2:], kk[..., : D // 2]), -1)
    return kk * cos + rot * sin, v.gather(2, g)


def main() -> None:
    from kvpress_b200 import native

    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="4096,32768,131072")
    ap.add_argument("--windows", default="64,512,2048")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    dev = "cuda:0"
    info = card()
    inv_freq = 1.0 / (500000.0 ** (torch.arange(0, D, 2, device=dev).float() / D))
    rows = []
    for S in map(int, a.sizes.split(",")):
        g = torch.Generator(device=dev).manual_seed(S)
        k = torch.randn(B, HKV, S, D, generator=g, device=dev).to(torch.bfloat16)
        v = torch.randn(B, HKV, S, D, generator=g, device=dev).to(torch.bfloat16)
        for w in map(int, a.windows.split(",")):
            q = torch.randn(B, HQ, w, D, generator=g, device=dev).to(torch.bfloat16)
            row = {"S": S, "w": w}
            row["score_ms"] = timed(lambda: native.finch_score(k, q, w), a.reps)
            row["tflops"] = 4 * B * HQ * w * S * D / (row["score_ms"] * 1e-3) / 1e12
            row["compress_ms"] = timed(lambda: native.finch_compress(k, v, q, w, RATIO, None, True, inv_freq), a.reps)
            row["compress_chunk4096_ms"] = timed(
                lambda: native.finch_compress(k, v, q, w, RATIO, CHUNK, True, inv_freq), a.reps)
            if w == 64:
                for name, L in (("chunkS", S), ("chunk5", 5)):
                    row[f"compress_{name}_ms"] = timed(
                        lambda: native.finch_compress(k, v, q, w, RATIO, L, True, inv_freq), a.reps)
            try:
                row["reference_ms"] = timed(lambda: reference(k, v, q, w, inv_freq), max(3, a.reps // 3))
            except torch.cuda.OutOfMemoryError:
                row["reference_ms"] = "oom"
            torch.cuda.empty_cache()
            rows.append(row)
            ref = row["reference_ms"]
            print(f"S {S:6d} w {w:4d}: score {row['score_ms']:.3f} ms ({row['tflops']:.0f} TFLOP/s of "
                  f"{DATASHEET_TFLOPS} data-sheet), compress {row['compress_ms']:.3f} ms, chunked "
                  f"{row['compress_chunk4096_ms']:.3f} ms, reference " +
                  (f"{ref:.3f} ms" if isinstance(ref, float) else ref) +
                  "".join(f", {n} {row[f'compress_{n}_ms']:.3f} ms" for n in ("chunkS", "chunk5")
                          if f"compress_{n}_ms" in row), flush=True)
    print(f"card: {info}")
    if a.json:
        Path(a.json).write_text(json.dumps({"card": info, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
