"""Times CAMPress's per-step accumulation and its compaction on the GPU, with the reference's restated in torch beside them.

    python scripts/bench_cam.py [--reps 20] [--json out.json]

At the Llama-3.1-8B layer shape (B 1, Hkv 8, Hq 32, D 128, bf16):
(a) the per-step path at S = 2,560, 32,768 and 131,072: `native.expected_attention_score` on the RoPE'd last query (the
    covariance-free scan) added into an fp32 capacity buffer, against the reference's step restated in torch
    (repeat_kv, matmul, fp32 softmax, cast, group mean, zero-pad cat, add into a bf16 running sum);
(b) compactions 2,560 -> 2,048 and 131,584 -> 2,048 (k 512, merge_budget 32): `native.cam_compress` against the
    reference's CAMPress.compress body restated in torch (three topk, argsort, searchsorted, gathers, bernoulli,
    scatter_add_, gathers).
Each is the median of `--reps` calls between CUDA events after two warm-up calls. The card's name and power limit are
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

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

B, HKV, HQ, D, TARGET, K, BUDGET = 1, 8, 32, 128, 2048, 512, 32


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


def reference_step(keys, q, running):  # q: [B, Hq, 1, D]
    """The reference's per-step accumulation: the last query's attention over the cache, added to a running sum in
    the cache dtype that grows by torch.cat."""
    G = HQ // HKV
    kr = keys[:, :, None].expand(B, HKV, G, *keys.shape[2:]).reshape(B, HQ, *keys.shape[2:])  # repeat_kv
    w = torch.matmul(q, kr.transpose(-2, -1)) / math.sqrt(D)
    w = torch.softmax(w, dim=-1, dtype=torch.float32).to(q.dtype)
    w = w.view(B, HKV, G, 1, -1).mean(2).squeeze(2)
    pad = torch.zeros(B, HKV, 1, dtype=running.dtype, device=running.device)
    running = torch.cat([running, pad], dim=-1)
    running += w
    return running


def reference_compress(scores, keys, values, attn, k, budget):
    """The reference's CAMPress.compress body after the base press's scores."""
    bsz, H, S, hd = keys.shape
    n_evict = S - TARGET
    mean = scores.mean(dim=1)
    ev = torch.sort(mean.topk(n_evict, dim=-1, largest=False).indices, dim=-1).values
    order = mean.gather(-1, ev).flip(-1).argsort(dim=-1, descending=True, stable=True)[:, :k]
    merge = torch.sort(ev.gather(-1, n_evict - 1 - order), dim=-1).values
    kept = torch.sort(mean.topk(TARGET, dim=-1).indices, dim=-1).values
    n = merge.shape[1]
    starts = torch.searchsorted(kept, merge, right=True)
    widx = starts.unsqueeze(-1) + torch.arange(budget, device=keys.device).view(1, 1, -1)
    valid = widx < TARGET
    tpos = kept.gather(1, widx.clamp(max=TARGET - 1).view(bsz, -1)).view(bsz, n, budget)
    actual = valid.sum(-1)
    wa = attn.gather(2, tpos.view(bsz, -1).unsqueeze(1).expand(-1, H, -1)).view(bsz, H, n, budget)
    mean_a = (wa * valid.view(bsz, 1, n, budget)).sum(-1) / actual.clamp(min=1).unsqueeze(1)
    p = attn.gather(2, merge.unsqueeze(1).expand(-1, H, -1)) / mean_a
    p = torch.where(torch.isnan(p), torch.zeros_like(p), p)
    p = torch.where(torch.isinf(p), torch.ones_like(p), p).clamp(0, 1)
    mask = torch.bernoulli(p)
    mv = values.gather(2, merge.view(bsz, 1, n, 1).expand(-1, H, -1, hd))
    scale = (mask / actual.unsqueeze(1)).unsqueeze(-1)
    contrib = (mv * scale).unsqueeze(3).expand(-1, -1, -1, budget, -1) * valid.view(bsz, 1, n, budget, 1)
    values = values.clone()
    values.scatter_add_(2, tpos.view(bsz, 1, n * budget, 1).expand(-1, H, -1, hd),
                        contrib.reshape(bsz, H, n * budget, hd))
    ke = kept.view(bsz, 1, TARGET, 1).expand(bsz, H, TARGET, hd)
    return keys.gather(2, ke).contiguous(), values.gather(2, ke).contiguous(), attn.gather(
        2, kept.unsqueeze(1).expand(bsz, H, -1)).contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    from kvpress_b200 import native
    from kvpress_b200.presses.cam_press import RunningAttention

    dev = "cuda"
    torch.manual_seed(0)
    results = {"card": card(), "step": [], "compress": []}
    for S in (2560, 32768, 131072):
        keys = torch.randn(B, HKV, S, D, device=dev, dtype=torch.bfloat16)
        q = torch.randn(B, HQ, D, device=dev, dtype=torch.bfloat16)
        state = RunningAttention(B, HKV, 2 * S, dev)
        state.add(torch.zeros(B, HKV, S - 1, device=dev))

        def ours():
            state.length = S - 1
            state.add(native.expected_attention_score(keys, keys, q, None, 0.0, 0, False))

        def scan_only():
            native.expected_attention_score(keys, keys, q, None, 0.0, 0, False)

        running = torch.zeros(B, HKV, S - 1, device=dev, dtype=torch.bfloat16)
        row = {"S": S, "ours_ms": timed(ours, args.reps), "scan_only_ms": timed(scan_only, args.reps),
               "reference_ms": timed(lambda: reference_step(keys, q.unsqueeze(2), running), args.reps)}
        results["step"].append(row)
        print(json.dumps({"step": row}), flush=True)
        del keys
    for S in (2560, 131584):
        keys = torch.randn(B, HKV, S, D, device=dev, dtype=torch.bfloat16)
        values = torch.randn(B, HKV, S, D, device=dev, dtype=torch.bfloat16)
        scores = torch.randn(B, HKV, S, device=dev).to(torch.bfloat16)
        attn = torch.rand(B, HKV, S, device=dev)
        out = torch.empty(B, HKV, TARGET, device=dev)
        u = torch.rand(B, HKV, K, device=dev)
        n_merge = min(K, S - TARGET)
        uu = u[..., :n_merge].contiguous()
        ours = lambda: native.cam_compress(scores, keys, values, attn, out, n_merge, BUDGET, uu, TARGET)  # noqa: E731
        row = {"S": S, "n_merge": n_merge, "ours_ms": timed(ours, args.reps)}
        try:
            attn_ref = attn.to(keys.dtype)  # the reference keeps its running sum in the cache dtype
            row["reference_ms"] = timed(lambda: reference_compress(scores, keys, values, attn_ref, K, BUDGET),
                                        args.reps)
        except torch.OutOfMemoryError:
            row["reference_ms"] = "oom"
        results["compress"].append(row)
        print(json.dumps({"compress": row}), flush=True)
    print(json.dumps(results))
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
