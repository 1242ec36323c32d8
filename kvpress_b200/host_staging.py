"""Host-buffer end-to-end path: K, V in pinned HOST memory -> compressed K', V' in pinned HOST memory.

Every (batch element, kv-head) row of the hot path is independent (SURVEY §8e), so a cache that lives in
host memory (offloaded caches, `transformers` OffloadedCache, the bench's `e2e` leg) does not have to cross
PCIe as one block before the first kernel starts. The cache is cut into chunks of `heads_per_chunk` kv-heads
and the three stages run on three streams,

    h2d stream     : chunk c+1  host -> device staging slot
    compute stream : chunk c    kvp_*_compress on the staging slot          (the C-ABI call)
    d2h stream     : chunk c-1  K', V' -> pinned host output

so the host link is busy in both directions at once and the kernels hide under the copies: the step costs
max(H2D, D2H) + one chunk of latency instead of H2D + compute + D2H.

`values_zero_copy=True` (scorers that never read V to score: Knorm, KeyDiff, SnapKV, StreamingLLM): V is not staged at
all — the compaction kernel reads the KEPT rows of V straight from the pinned host buffer over PCIe (UVA), so
only n_kept/S of V crosses the link.

torch is used for memory, streams and events only; the compute is the C-ABI library. No CPU compute path.
"""
from __future__ import annotations

from typing import Optional

import torch

from kvpress_b200 import native

_STREAMS: dict = {}
N_SLOTS = 3


def _streams(device: torch.device):
    key = (device.type, device.index)
    if key not in _STREAMS:
        _STREAMS[key] = tuple(torch.cuda.Stream(device=device) for _ in range(3))
    return _STREAMS[key]


def _require_pinned(name: str, t: torch.Tensor):
    if t.is_cuda or not t.is_pinned():
        raise RuntimeError(f"{name} must be a pinned host tensor (torch.Tensor.pin_memory()), got {t.device}")
    if t.dim() != 4 or not t.is_contiguous():
        raise RuntimeError(f"{name} must be a contiguous [B, Hkv, S, D] tensor")


def _run_chunk(scorer: str, k, v, n_kept: int, b: int, hq0: int, hq1: int, params: dict):
    if scorer == "knorm":
        return native.knorm_compress(k, v, n_kept, _pinned_values=not v.is_cuda)[:2]
    if scorer == "keydiff":
        return native.keydiff_compress(k, v, n_kept, _pinned_values=not v.is_cuda)[:2]
    if scorer == "streaming":
        return native.streaming_compress(k, v, n_kept, params.get("n_sink", 4), _pinned_kv=not v.is_cuda)[:2]
    if scorer == "snapkv":
        q = params["q_window"][b:b + 1, hq0:hq1]
        return native.snapkv_compress(k, v, q, params.get("window", q.shape[2]), params.get("kernel_size", 5), n_kept,
                                      _pinned_values=not v.is_cuda)[:2]
    if scorer == "expected_attention":
        cov = params.get("cov")
        return native.expected_attention_compress(
            k, v, params["mu"][b:b + 1, hq0:hq1], None if cov is None else cov[b:b + 1, hq0:hq1], params.get("epsilon", 0.0),
            params.get("n_sink", 4), params.get("use_vnorm", True), n_kept)[:2]
    raise ValueError(f"unknown scorer {scorer!r}")


def compress_host(scorer: str, keys_host: torch.Tensor, values_host: torch.Tensor, n_kept: int, *,
                  device="cuda", out_keys: Optional[torch.Tensor] = None, out_values: Optional[torch.Tensor] = None,
                  heads_per_chunk: int = 1, values_zero_copy: Optional[bool] = None, num_q_heads: Optional[int] = None,
                  **params):
    """ScorerPress.compress (scorer_press.py:76-102) for a cache held in pinned host memory.

    scorer: "knorm" | "keydiff" | "streaming" | "snapkv" | "expected_attention"; params are the scorer's device-resident
    small operands (q_window / mu, cov, ...) with all Hq heads — they are sliced per chunk here.
    Returns pinned host (K', V') of shape [B, Hkv, n_kept, D], rows in ascending position order. The call
    returns after the three streams have drained (outputs are ready to read on the host)."""
    _require_pinned("keys_host", keys_host)
    _require_pinned("values_host", values_host)
    device = torch.device(device)
    if device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    B, H, S, D = keys_host.shape
    if out_keys is None:
        out_keys = torch.empty((B, H, n_kept, D), dtype=keys_host.dtype).pin_memory()
    if out_values is None:
        out_values = torch.empty((B, H, n_kept, D), dtype=keys_host.dtype).pin_memory()
    _require_pinned("out_keys", out_keys)
    _require_pinned("out_values", out_values)
    if n_kept == 0:
        return out_keys, out_values
    if values_zero_copy is None:
        values_zero_copy = False
    if values_zero_copy and scorer == "expected_attention":
        raise RuntimeError("values_zero_copy needs a scorer that does not read V to score (Knorm, KeyDiff, SnapKV, "
                           "StreamingLLM)")
    Hq = num_q_heads or {"snapkv": lambda: params["q_window"].shape[1],
                         "expected_attention": lambda: params["mu"].shape[1]}.get(scorer, lambda: H)()
    G = Hq // H
    nh = max(1, min(heads_per_chunk, H))
    chunks = [(b, h0, min(h0 + nh, H)) for b in range(B) for h0 in range(0, H, nh)]
    streaming_zero_copy = values_zero_copy and scorer == "streaming"  # K is only gathered too

    s_h2d, s_cmp, s_d2h = _streams(device)
    caller = torch.cuda.current_stream(device)
    with torch.cuda.device(device):
        fork = torch.cuda.Event()
        fork.record(caller)
        for s in (s_h2d, s_cmp, s_d2h):
            s.wait_event(fork)
        n_slots = min(N_SLOTS, len(chunks))
        with torch.cuda.stream(s_h2d):
            k_slots = None if streaming_zero_copy else [
                torch.empty((1, nh, S, D), dtype=keys_host.dtype, device=device) for _ in range(n_slots)]
            v_slots = None if values_zero_copy else [torch.empty_like(k) for k in k_slots]
        slot_free = [None] * n_slots  # compute-done event of the chunk that last used the slot
        keep_alive, last_d2h = [], None
        for c, (b, h0, h1) in enumerate(chunks):
            slot, n = c % n_slots, h1 - h0
            k_src, v_src = keys_host[b:b + 1, h0:h1], values_host[b:b + 1, h0:h1]
            with torch.cuda.stream(s_h2d):
                if slot_free[slot] is not None:
                    s_h2d.wait_event(slot_free[slot])
                k_dev = k_src if streaming_zero_copy else k_slots[slot][:, :n].copy_(k_src, non_blocking=True)
                v_dev = v_src if values_zero_copy else v_slots[slot][:, :n].copy_(v_src, non_blocking=True)
                staged = torch.cuda.Event()
                staged.record(s_h2d)
            with torch.cuda.stream(s_cmp):
                s_cmp.wait_event(staged)
                k2, v2 = _run_chunk(scorer, k_dev, v_dev, n_kept, b, h0 * G, h1 * G, params)
                done = torch.cuda.Event()
                done.record(s_cmp)
                slot_free[slot] = done
            with torch.cuda.stream(s_d2h):
                s_d2h.wait_event(done)
                out_keys[b:b + 1, h0:h1].copy_(k2, non_blocking=True)
                out_values[b:b + 1, h0:h1].copy_(v2, non_blocking=True)
                last_d2h = torch.cuda.Event()
                last_d2h.record(s_d2h)
            keep_alive.append((k2, v2))  # allocated on s_cmp, read on s_d2h: hold until drained
        caller.wait_event(last_d2h)
        caller.wait_stream(s_cmp)
        caller.wait_stream(s_h2d)
        last_d2h.synchronize()
        s_cmp.synchronize()
    del keep_alive, k_slots, v_slots
    return out_keys, out_values
