"""Scores for cache shapes the tensor-core scorers do not instantiate (GPU, torch / cuBLAS GEMMs).

The tensor-core (wgmma) SnapKV and ExpectedAttention kernels keep their query block / covariance resident in shared memory
and exist for head_dim 64 and 128, at most 8 query heads per kv head and (for SnapKV) at most 512 window-query rows
per kv head. Phi-3 (head_dim 96) and Gemma-3 (head_dim 256) fall outside. For those shapes only the SCORE stage
is evaluated here with plain library GEMMs on the GPU, in fp32 with one rounding to the cache dtype — the same
definition the kernels implement ("fp32 evaluation of the reference formula, rounded once", DESIGN.md §2) — and the
result goes through the sm_90a selection + compaction kernels like any caller-supplied score tensor
(`native.scores_compress`). Nothing here runs on the CPU; CPU tensors are refused like everywhere else.

Every GEMM operand is a 16-bit value (the cache's, or the model's queries) widened to fp32, and the scales (1/sqrt(d), 1/(2d), the attention
`scaling`) multiply the fp32 GEMM results, never an operand. fp32 matmuls follow the process-wide
`torch.backends.cuda.matmul.fp32_precision`: under "tf32" (what `torch.set_float32_matmul_precision("high")` selects)
cuBLAS rounds its operands to 10 mantissa bits. A scaled operand would lose up to 2^-11 of itself there, which the
softmax turns into several fp16 ulps of error at logits near 20. A 16-bit value fits TF32 exactly, and its products are
exact and summed in fp32, so the result keeps the contract whatever the caller has set. The setting itself is never
touched here: it is global to the process, shared between threads, and the caller's to choose.

Formulas: SnapKV `kvpress/presses/snapkv_press.py:41-105`, ExpectedAttention
`kvpress/presses/expected_attention_press.py:136-165`, CriticalKV `kvpress/presses/criticalkv_press.py:57-92` (head_dim
other than 64 / 128), ObservedAttention `kvpress/presses/observed_attention_press.py` (head_dim other than 64 / 128, more
than 8 query heads per kv head), NonCausalAttention `kvpress/presses/non_causal_attention_press.py` (head_dim other than
64 / 128, more than 8 query heads per kv head, chunk sizes other than 128 / 256).
"""
from __future__ import annotations

import logging
import math

import torch
import torch.nn.functional as F

logger = logging.getLogger(__name__)
_warned: set = set()

TENSOR_CORE_HEAD_DIMS = (64, 128)
MAX_GROUP = 8
MAX_SNAP_QUERY_ROWS = 512


def snapkv_on_tensor_cores(head_dim: int, group: int, window: int) -> bool:
    """Shapes `kvp_snapkv_*` instantiates (csrc/snapkv.cu launch_snap_d)."""
    return head_dim in TENSOR_CORE_HEAD_DIMS and 1 <= group * window <= MAX_SNAP_QUERY_ROWS


def expected_attention_on_tensor_cores(head_dim: int, group: int, has_cov: bool) -> bool:
    """Shapes `kvp_expected_attention_*` instantiates (csrc/expected_attention.cu launch_ea_t): the covariance-free
    scan takes any head_dim, the covariance path head_dim 64 / 128; both at most 8 query heads per kv head."""
    return group <= MAX_GROUP and (not has_cov or head_dim in TENSOR_CORE_HEAD_DIMS)


def criticalkv_on_tensor_cores(head_dim: int) -> bool:
    """Shapes `kvp_criticalkv_*` instantiates (csrc/criticalkv.cu): head_dim 64 / 128, any group size and hidden size."""
    return head_dim in TENSOR_CORE_HEAD_DIMS


def observed_attention_on_tensor_cores(head_dim: int, group: int) -> bool:
    """Shapes `kvp_observed_attention_*` instantiates (csrc/observed_attention.cu launch_obs_d): head_dim 64 / 128, at
    most 8 query heads per kv head."""
    return head_dim in TENSOR_CORE_HEAD_DIMS and 1 <= group <= MAX_GROUP


def non_causal_attention_on_tensor_cores(head_dim: int, group: int, chunk_size: int) -> bool:
    """Shapes `kvp_non_causal_attention_*` instantiates (csrc/non_causal_attention.cu launch_nca_d): head_dim 64 / 128,
    chunk_size 128 / 256, at most 8 query heads per kv head."""
    return head_dim in TENSOR_CORE_HEAD_DIMS and chunk_size in (128, 256) and 1 <= group <= MAX_GROUP


def _note(what: str, keys: torch.Tensor, group: int) -> None:
    key = (what, keys.shape[-1], group)
    if key not in _warned:
        _warned.add(key)
        logger.warning(f"{what}: head_dim {keys.shape[-1]} / {group} query heads per kv head is outside the tensor-core "
                       "scorer instantiations; scoring with cuBLAS GEMMs, selection + compaction stay on the "
                       "sm_90a kernels")


def _require_cuda(keys: torch.Tensor) -> None:
    if not keys.is_cuda:
        raise RuntimeError(f"kvpress_b200 runs on CUDA tensors only; got keys on {keys.device}. There is no CPU path.")


def _pad_forced(scores: torch.Tensor, n_front: int, n_back: int) -> torch.Tensor:
    """Forced-keep positions carry max + 1 over the whole tensor (snapkv_press.py:103, expected_attention_press.py:163),
    formed on the device (no host sync) and rounded once to the score dtype."""
    sentinel = (scores.max().float() + 1).to(scores.dtype)
    B, H, _ = scores.shape
    parts = []
    if n_front:
        parts.append(sentinel.expand(B, H, n_front))
    parts.append(scores)
    if n_back:
        parts.append(sentinel.expand(B, H, n_back))
    return torch.cat(parts, dim=-1)


def snapkv_scores(keys: torch.Tensor, q_window: torch.Tensor, window: int, kernel_size: int,
                  chunk: int = 16384) -> torch.Tensor:
    """keys [B,Hkv,S,D], RoPE'd window queries [B,Hq,w,D] -> scores [B,Hkv,S] in the cache dtype."""
    _require_cuda(keys)
    B, Hkv, S, D = keys.shape
    G, w = q_window.shape[1] // Hkv, window
    _note("SnapKV", keys, G)
    q = q_window.float().reshape(B, Hkv, G * w, D)
    logits = torch.empty((B, Hkv, G * w, S), dtype=torch.float32, device=keys.device)
    for s0 in range(0, S, chunk):  # fp32 copies of K one slab at a time
        s1 = min(S, s0 + chunk)
        torch.matmul(q, keys[:, :, s0:s1].float().transpose(-1, -2), out=logits[..., s0:s1])
    logits.mul_(1.0 / math.sqrt(D))
    # inside the window query i (position S - w + i) does not see key S - w + j for j > i
    future = torch.ones((w, w), dtype=torch.bool, device=keys.device).triu(1)
    logits.view(B, Hkv, G, w, S)[..., S - w:].masked_fill_(future, float("-inf"))
    prob = torch.softmax(logits, dim=-1)
    del logits
    col = prob[..., : S - w].mean(dim=2)                               # mean over the window and the group
    col = F.avg_pool1d(col, kernel_size=kernel_size, padding=kernel_size // 2, stride=1)  # zero pad, always / kernel
    return _pad_forced(col.to(keys.dtype), 0, w)


def expected_attention_scores(keys: torch.Tensor, values: torch.Tensor, mu: torch.Tensor, cov, epsilon: float,
                              n_sink: int, use_vnorm: bool, chunk: int = 4096) -> torch.Tensor:
    """keys/values [B,Hkv,S,D], mu [B,Hq,D], cov [B,Hq,D,D] or None -> scores [B,Hkv,S] in the cache dtype."""
    _require_cuda(keys)
    B, Hkv, S, D = keys.shape
    G = mu.shape[1] // Hkv
    _note("ExpectedAttention", keys, G)
    L = S - n_sink
    mu_f = mu.to(keys.dtype).float().reshape(B, Hkv, G, D)                    # operands in the cache dtype,
    cov_f = None if cov is None else cov.to(keys.dtype).float().reshape(B, Hkv, G, D, D)  # like the C ABI
    logits = torch.empty((B, Hkv, G, L), dtype=torch.float32, device=keys.device)
    for s0 in range(0, L, chunk):
        s1 = min(L, s0 + chunk)
        k = keys[:, :, n_sink + s0:n_sink + s1].float()               # [B,Hkv,c,D]
        part = torch.matmul(mu_f, k.transpose(-1, -2)) * (1.0 / math.sqrt(D))    # mu.k / sqrt(d)
        if cov_f is not None:                                          # + k^T Sigma k / 2d
            y = torch.matmul(k.unsqueeze(2), cov_f)                    # [B,Hkv,G,c,D]
            part = part + (y * k.unsqueeze(2)).sum(dim=-1) * (0.5 / D)
        logits[..., s0:s1] = part
    score = torch.softmax(logits, dim=-1).mean(dim=2)                  # [B,Hkv,L]
    if use_vnorm:
        vn = torch.empty((B, Hkv, L), dtype=torch.float32, device=keys.device)
        for s0 in range(0, L, 4 * chunk):
            s1 = min(L, s0 + 4 * chunk)
            vn[..., s0:s1] = values[:, :, n_sink + s0:n_sink + s1].float().norm(dim=-1)
        score = (score + epsilon) * vn
    return _pad_forced(score.to(keys.dtype), n_sink, 0)


def criticalkv_scores(base_scores: torch.Tensor, values: torch.Tensor, wo: torch.Tensor, epsilon: float, n_first: int,
                      chunk: int = 4096) -> torch.Tensor:
    """CriticalKV scores [B,Hkv,S] in the cache dtype from the wrapped press's scores, values [B,Hkv,S,D] and
    o_proj.weight [hidden, Hq*D]: one query head and one slab of positions at a time in fp32, rounded once; the
    n_first best base scores of every row get finfo.max through the sm_90a selection."""
    from kvpress_b200 import native

    _require_cuda(values)
    B, Hkv, S, D = values.shape
    Hq = wo.shape[1] // D
    G = Hq // Hkv
    _note("CriticalKV", values, G)
    base = base_scores.to(values.dtype)
    w = wo.to(values.dtype).float()
    norm = torch.zeros((B, Hkv, S), dtype=torch.float32, device=values.device)
    for h in range(Hq):
        w_h = w[:, h * D:(h + 1) * D]                                   # [hidden, D]
        for s0 in range(0, S, chunk):
            s1 = min(S, s0 + chunk)
            v = values[:, h // G, s0:s1].float()                        # [B, c, D]
            norm[:, h // G, s0:s1] += torch.matmul(v, w_h.T).abs().sum(dim=-1)
    scores = ((base.float() + epsilon) * (norm / G)).to(values.dtype)
    if n_first > 0:
        first = native.scores_select(base, n_first).long()
        scores.scatter_(-1, first, torch.finfo(scores.dtype).max)
    return scores


def observed_attention_scores(keys: torch.Tensor, q: torch.Tensor, scaling: float,
                              max_logits: int = 1 << 27) -> torch.Tensor:
    """keys [B,Hkv,S,D], RoPE'd queries [B,Hq,n_q,D] of positions S - n_q .. S - 1 -> H2O scores [B,Hkv,S] in the cache
    dtype: (1/G) sum over the group's query rows of the causal softmax(scaling q.k), / (S - s) rounded to the cache
    dtype. Two passes over blocks of query rows in fp32: the row log-sum-exp, then the column sums; at most one block
    of logits ([B, Hq, rows, S], at most `max_logits` elements) exists at a time."""
    _require_cuda(keys)
    B, Hkv, S, D = keys.shape
    Hq, n_q = q.shape[1], q.shape[2]
    G, off = Hq // Hkv, S - n_q
    _note("ObservedAttention", keys, G)
    block = max(1, max_logits // (B * Hq * S))
    k = keys.float().unsqueeze(2)                                      # [B,Hkv,1,S,D]
    qf = q.to(keys.dtype).float().reshape(B, Hkv, G, n_q, D)
    pos = torch.arange(S, device=keys.device)

    def logits(i0: int, i1: int) -> torch.Tensor:                      # [B,Hkv,G,i1-i0,S], causal
        y = torch.matmul(qf[:, :, :, i0:i1], k.transpose(-1, -2)).mul_(scaling)
        rows = torch.arange(off + i0, off + i1, device=keys.device)
        return y.masked_fill_(pos[None, :] > rows[:, None], float("-inf"))

    lse = torch.empty((B, Hkv, G, n_q, 1), dtype=torch.float32, device=keys.device)
    for i0 in range(0, n_q, block):
        i1 = min(n_q, i0 + block)
        lse[:, :, :, i0:i1] = torch.logsumexp(logits(i0, i1), dim=-1, keepdim=True)
    col = torch.zeros((B, Hkv, S), dtype=torch.float32, device=keys.device)
    for i0 in range(0, n_q, block):
        i1 = min(n_q, i0 + block)
        col += torch.exp(logits(i0, i1) - lse[:, :, :, i0:i1]).sum(dim=(2, 3))
    div = torch.arange(S, 0, -1, device=keys.device).to(keys.dtype).float()
    return (col / (G * div)).to(keys.dtype)


def non_causal_attention_scores(keys: torch.Tensor, values: torch.Tensor, q: torch.Tensor, chunk_size: int,
                                max_logits: int = 1 << 27) -> torch.Tensor:
    """keys / values [B,Hkv,S,D], RoPE'd queries [B,Hq,S,D] -> NonCausalAttnPress z-scores [B,Hkv,S] in the cache
    dtype, by the definition of include/kvpress_b200.h (kvp_non_causal_attention_score): fp32 over blocks of chunks (at
    most `max_logits` logits at a time), the padded last chunk as the reference pads it, one rounding."""
    _require_cuda(keys)
    B, Hkv, S, D = keys.shape
    G, cs = q.shape[1] // Hkv, int(chunk_size)
    _note("NonCausalAttention", keys, G)
    n_chunks = -(-S // cs)
    pad = n_chunks * cs - S
    kf = F.pad(keys.float(), (0, 0, 0, pad)).view(B, Hkv, 1, n_chunks, cs, D)
    qf = F.pad(q.to(keys.dtype).float(), (0, 0, 0, pad)).view(B, Hkv, G, n_chunks, cs, D)
    colsum = torch.empty((B, Hkv, n_chunks, cs), dtype=torch.float32, device=keys.device)
    block = max(1, max_logits // (B * Hkv * G * cs * cs))
    for c0 in range(0, n_chunks, block):
        c1 = min(n_chunks, c0 + block)
        y = torch.matmul(qf[:, :, :, c0:c1], kf[:, :, :, c0:c1].transpose(-1, -2))   # [B,Hkv,G,c,cs,cs]
        if pad and c1 == n_chunks:   # padded query rows: uniform over the chunk; padded keys stay at logit 0
            y[:, :, :, -1, cs - pad:] = 0
        colsum[:, :, c0:c1] = torch.softmax(y, dim=-1).sum(dim=-2).mean(dim=2)
        del y
    x = colsum.view(B, Hkv, n_chunks * cs)[..., :S] * values.float().norm(dim=-1)
    pooled = F.avg_pool1d(x, kernel_size=3, padding=1, stride=1)
    return ((pooled - pooled.mean()) / pooled.std().clamp_min(1e-6)).to(keys.dtype)
