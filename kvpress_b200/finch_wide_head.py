"""FinchPress scores for cache shapes the tensor-core kernels do not instantiate (GPU, torch / cuBLAS GEMMs).

`kvp_finch_*` exists for head_dim 64 / 128 and at most 8 query heads per kv head (csrc/finch.cu launch_finch_d). For
other shapes the SCORE stage is evaluated here the way wide_head_scores.py evaluates the other scorers (fp32 from the
16-bit operands, one rounding to the cache dtype; see its docstring for the TF32 argument), and the selection runs on
the sm_90a kernels (`native.scores_compress`, `scores_compress_rerotate`, `scores_compress_chunked`). Formula:
`kvpress/presses/finch_press.py`, with the weights c_i exact as in include/kvpress_b200.h.
"""
from __future__ import annotations

import math

import torch

from kvpress_b200.wide_head_scores import MAX_GROUP, TENSOR_CORE_HEAD_DIMS, _note, _pad_forced, _require_cuda


def finch_on_tensor_cores(head_dim: int, group: int) -> bool:
    """Shapes `kvp_finch_*` instantiates: head_dim 64 / 128, at most 8 query heads per kv head, any window."""
    return head_dim in TENSOR_CORE_HEAD_DIMS and 1 <= group <= MAX_GROUP


def finch_scores(keys: torch.Tensor, q_window: torch.Tensor, window: int, normalize: bool = True,
                 max_logits: int = 1 << 27) -> torch.Tensor:
    """keys [B,Hkv,S,D], RoPE'd window queries [B,Hq,w,D] of positions S - w .. S - 1 -> FinchPress scores [B,Hkv,S]
    in the cache dtype: 1/(G w) sum over the group's window rows of c_i softmax(q.k / sqrt(D)) (causal inside the
    window, c_i = S - w + i exact, or 1 without normalize) at the context positions, the window padded with the
    max + 1 sentinel. Two passes over blocks of window rows in fp32: the row log-sum-exp, then the weighted column sums
    of the context; at most one block of logits ([B, Hq, rows, S], at most `max_logits` elements) exists at a time,
    never the whole [B, Hq, w, S]."""
    _require_cuda(keys)
    B, Hkv, S, D = keys.shape
    Hq, w = q_window.shape[1], window
    G, off = Hq // Hkv, S - window
    _note("Finch", keys, G)
    block = max(1, max_logits // (B * Hq * S))
    k = keys.float().unsqueeze(2)                                      # [B,Hkv,1,S,D]
    qf = q_window.to(keys.dtype).float().reshape(B, Hkv, G, w, D)
    pos = torch.arange(S, device=keys.device)
    scale = 1.0 / math.sqrt(D)

    def logits(i0: int, i1: int) -> torch.Tensor:                      # [B,Hkv,G,i1-i0,S], causal
        y = torch.matmul(qf[:, :, :, i0:i1], k.transpose(-1, -2)).mul_(scale)
        rows = torch.arange(off + i0, off + i1, device=keys.device)
        return y.masked_fill_(pos[None, :] > rows[:, None], float("-inf"))

    lse = torch.empty((B, Hkv, G, w, 1), dtype=torch.float32, device=keys.device)
    for i0 in range(0, w, block):
        i1 = min(w, i0 + block)
        lse[:, :, :, i0:i1] = torch.logsumexp(logits(i0, i1), dim=-1, keepdim=True)
    col = torch.zeros((B, Hkv, off), dtype=torch.float32, device=keys.device)
    for i0 in range(0, w, block):
        i1 = min(w, i0 + block)
        p = torch.exp(logits(i0, i1)[..., :off] - lse[:, :, :, i0:i1])
        if normalize:
            p.mul_(torch.arange(off + i0, off + i1, device=keys.device, dtype=torch.float32)[:, None])
        col += p.sum(dim=(2, 3))
    return _pad_forced((col / (G * w)).to(keys.dtype), 0, w)
