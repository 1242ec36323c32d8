"""A float64 stand-in for native.finch_score / finch_compress / scores_compress_chunked: the definition of
include/kvpress_b200.h (kvp_finch_*) evaluated in float64 and rounded once to the cache dtype, the window forced, the
per-chunk top-k with ties to the lowest position in ascending order, and the kept keys re-rotated by (j - s) inv_freq
in float64. Pure torch on any device: the host tests put it in place of the kernels, the GPU tests compare with it."""
import math

import torch

from kvpress_b200 import native


def context64(keys: torch.Tensor, q_window: torch.Tensor, window: int, normalize: bool = True) -> torch.Tensor:
    """float64 [B, Hkv, S - w]: 1/(G w) sum_g sum_i c_i softmax(q.k / sqrt(D)), causal inside the window."""
    B, H, S, D = keys.shape
    G, w = q_window.shape[1] // H, window
    y = torch.einsum("bhgid,bhsd->bhgis", q_window.double().reshape(B, H, G, w, D), keys.double()) / math.sqrt(D)
    rpos = torch.arange(S - w, S, device=keys.device)
    y.masked_fill_(torch.arange(S, device=keys.device)[None, :] > rpos[:, None], float("-inf"))
    p = torch.softmax(y, dim=-1)[..., : S - w]
    if normalize:
        p = p * rpos.double()[:, None]
    return p.sum(dim=(2, 3)) / (G * w)


def finch_score64(keys, q_window, window: int, normalize: bool = True) -> torch.Tensor:
    """native.finch_score's contract: the context scores rounded once, the window at the call's max + 1."""
    ctx = context64(keys, q_window, window, normalize).to(keys.dtype)
    sentinel = (ctx.max().double() + 1).to(keys.dtype)
    return torch.cat([ctx, sentinel.expand(*ctx.shape[:2], window)], dim=-1)


def select(scores: torch.Tensor, window: int, chunk_length, ratio: float) -> torch.Tensor:
    """int64 [B, H, n_kept]: per chunk (the whole row when chunk_length is None / 0) its best positions, the last
    `window` positions forced, ties to the lowest position, ascending."""
    S = scores.shape[-1]
    s = scores.double().clone()
    if window:
        s[..., S - window:] = float("inf")
    L = chunk_length or S
    out = []
    for lo in range(0, S, L):
        hi = min(S, lo + L)
        n = int(S * (1 - ratio)) if not chunk_length else max(1, int((hi - lo) * (1 - ratio)))
        order = torch.sort(-s[..., lo:hi], dim=-1, stable=True).indices[..., :n]
        out.append(order.sort(dim=-1).values + lo)
    return torch.cat(out, dim=-1)


def gather(x: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    return x.gather(2, idx.unsqueeze(-1).expand(-1, -1, -1, x.shape[-1]))


def rerotate64(keys: torch.Tensor, idx: torch.Tensor, inv_freq: torch.Tensor) -> torch.Tensor:
    """keys[idx] rotated by (j - idx_j) inv_freq, in float64, rounded once to the cache dtype."""
    D = keys.shape[-1]
    k = gather(keys, idx).double()
    delta = (torch.arange(idx.shape[-1], device=keys.device) - idx).double()
    ang = delta[..., None] * inv_freq.to(keys.device).double()
    cos, sin = torch.cat((ang.cos(),) * 2, -1), torch.cat((ang.sin(),) * 2, -1)
    rot = torch.cat((-k[..., D // 2:], k[..., : D // 2]), -1)
    return (k * cos + rot * sin).to(keys.dtype)


def _outputs(scores, keys, values, idx, inv_freq, return_indices):
    k_out = rerotate64(keys, idx, inv_freq) if inv_freq is not None else gather(keys, idx)
    return k_out, gather(values, idx), idx.to(torch.int32) if return_indices else None


def finch_compress64(keys, values, q_window, window: int, compression_ratio: float, chunk_length=None,
                     normalize: bool = True, inv_freq=None, return_indices: bool = False, return_scores: bool = False):
    scores = finch_score64(keys, q_window, window, normalize)
    idx = select(scores, window, chunk_length, compression_ratio)
    return (*_outputs(scores, keys, values, idx, inv_freq, return_indices), scores if return_scores else None)


def scores_compress_chunked64(scores, keys, values, compression_ratio: float, chunk_length: int, inv_freq=None,
                              return_indices: bool = False):
    idx = select(scores.to(keys.dtype), 0, chunk_length, compression_ratio)
    return _outputs(scores, keys, values, idx, inv_freq, return_indices)


def install(monkeypatch):
    """The stand-ins in place of the kernels, and every shape routed to them (the tiny models have head_dim 16)."""
    from kvpress_b200 import finch_wide_head

    monkeypatch.setattr(native, "finch_score", finch_score64)
    monkeypatch.setattr(native, "finch_compress", finch_compress64)
    monkeypatch.setattr(native, "scores_compress_chunked", scores_compress_chunked64)
    monkeypatch.setattr(finch_wide_head, "finch_on_tensor_cores", lambda *a: True)
