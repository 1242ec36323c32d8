"""Float64 restatement of the LagKV score and oracle-backed stand-ins for `native.lagkv_score` / `native.lagkv_compress`,
used by the LagKV tests next to tests/cpu_backend.py: the same contract (float64 evaluation rounded once, ascending
positions, lowest-position ties). Pure torch: they run on CPU or CUDA tensors."""
import torch

from tests.cpu_backend import select_gather


def is_short(S: int, n_sink: int, lag_size: int) -> bool:
    return S < n_sink + 2 * lag_size


def sigma64(x: torch.Tensor, n_sink: int, lag_size: int) -> torch.Tensor:
    """sigma[b, j, c, s] of every scored partition c (include/kvpress_b200.h, kvp_lagkv_score) in float64: the
    unbiased std over the channels of (x - lo) / (hi - lo), lo / hi the per-channel min / max of partition c + 1."""
    B, H, S, D = x.shape
    P = (S - n_sink) // lag_size
    t = x[:, :, n_sink:n_sink + P * lag_size].double().reshape(B, H, P, lag_size, D)
    lo = t[:, :, 1:].amin(dim=-2, keepdim=True)
    hi = t[:, :, 1:].amax(dim=-2, keepdim=True)
    return ((t[:, :, :-1] - lo) / (hi - lo)).std(dim=-1)


def combined64(keys, values, n_sink: int, lag_size: int) -> torch.Tensor:
    """c = (softmax(sigma_k) + softmax(sigma_v)) / 2 over each scored partition, float64 [B, Hkv, P - 1, L]."""
    ak = sigma64(keys, n_sink, lag_size).softmax(dim=-1)
    av = sigma64(values, n_sink, lag_size).softmax(dim=-1)
    return (ak + av) / 2


def ranks(c: torch.Tensor) -> torch.Tensor:
    """r(s) = #{t : c(t) < c(s)} + #{t < s : c(t) = c(s)} along the last dim, NaN above every number and equal to NaN:
    the inverse of a stable ascending sort."""
    return torch.sort(c, dim=-1, stable=True).indices.argsort(dim=-1)


def lagkv_scores64(keys, values, n_sink: int, lag_size: int, cross_scoring: bool) -> torch.Tensor:
    """The definition before the final rounding to the cache dtype: float64 [B, Hkv, S]. Ranks and the short-cache ramp
    are the fp32 quotients of the definition, exact in float64."""
    B, H, S, _ = keys.shape
    out = torch.ones((B, H, S), dtype=torch.float64, device=keys.device)
    if is_short(S, n_sink, lag_size):
        if S > n_sink:
            ramp = torch.arange(S - n_sink, device=keys.device, dtype=torch.float32) / float(S - n_sink)
            out[..., n_sink:] = ramp.double()
        return out
    c = combined64(keys, values, n_sink, lag_size)
    if not cross_scoring:
        c = (ranks(c).to(torch.float32) / float(lag_size)).double()
    P = (S - n_sink) // lag_size
    out[..., n_sink:n_sink + (P - 1) * lag_size] = c.reshape(B, H, -1)
    return out


def lagkv_score(keys, values, n_sink, lag_size, cross_scoring):
    """lagkv_scores64 rounded once to the cache dtype."""
    return lagkv_scores64(keys, values, n_sink, lag_size, cross_scoring).to(keys.dtype)


def lagkv_compress(keys, values, n_sink, lag_size, cross_scoring, n_kept, return_indices=False, return_scores=False):
    scores = lagkv_score(keys, values, n_sink, lag_size, cross_scoring)
    return select_gather(scores, keys, values, n_kept, return_indices, return_scores)


def install(monkeypatch):
    from kvpress_b200 import native

    monkeypatch.setattr(native, "lagkv_score", lagkv_score)
    monkeypatch.setattr(native, "lagkv_compress", lagkv_compress)
