"""Float64 restatement of the CUR score and oracle-backed stand-ins for `native.cur_score` / `native.cur_compress`, used
by the CUR tests next to tests/cpu_backend.py: the same contract (float64 evaluation rounded once, ascending positions,
lowest-position ties). Pure torch: they run on CPU or CUDA tensors."""
import torch

from tests.cpu_backend import select_gather

LEVERAGE_TYPES = ("key", "value", "kv_avg", "kv_product")


def share64(x: torch.Tensor, window: int, G=None) -> torch.Tensor:
    """p[b, j, s] (include/kvpress_b200.h, kvp_cur_score) in float64: the squared norm of row s (of its projection by G),
    divided by the sum over its window of `window` positions; the last window sums its real positions only.
    window 0: not divided."""
    x = x.double()
    a = (x if G is None else x @ G.double()).square().sum(dim=-1)
    if window > 0:
        S = a.shape[-1]
        pad = (window - S % window) % window
        a = torch.nn.functional.pad(a, (0, pad)).unflatten(-1, (-1, window))
        a = (a / a.sum(dim=-1, keepdim=True)).flatten(-2)[..., :S]
    return a


def combined64(keys, values, leverage_type: str, window: int, G=None) -> torch.Tensor:
    """u[b, j, s] in float64."""
    if leverage_type == "key":
        return share64(keys, window, G)
    if leverage_type == "value":
        return share64(values, window, G)
    if leverage_type == "kv_avg":
        return (share64(keys, window, G) + share64(values, window, G)) / 2
    if leverage_type == "kv_product":
        return share64(keys, window, G) * share64(values, window, G)
    raise ValueError("Unknown leverage type: choose from 'kv_avg', 'key', 'value' or 'kv_product'")


def cur_scores64(keys, values, num_sinks: int, leverage_type: str, window: int, G=None) -> torch.Tensor:
    """The definition before the final rounding to the cache dtype: float64 [B, Hkv, S]."""
    assert num_sinks >= 0 and window >= 0
    u = combined64(keys, values, leverage_type, window, G)
    scores = u / u.sum(dim=-1, keepdim=True)
    scores[..., :num_sinks] = 1.0
    return scores


def cur_score(keys, values, num_sinks, leverage_type, local_window_size, G=None):
    """cur_scores64 rounded once to the cache dtype."""
    return cur_scores64(keys, values, num_sinks, leverage_type, local_window_size, G).to(keys.dtype)


def cur_compress(keys, values, num_sinks, leverage_type, local_window_size, G, n_kept, return_indices=False,
                 return_scores=False):
    scores = cur_score(keys, values, num_sinks, leverage_type, local_window_size, G)
    return select_gather(scores, keys, values, n_kept, return_indices, return_scores)


def install(monkeypatch):
    from kvpress_b200 import native

    monkeypatch.setattr(native, "cur_score", cur_score)
    monkeypatch.setattr(native, "cur_compress", cur_compress)
