"""CURPress: approximate leverage scores of the keys and the values (CurDKV, https://arxiv.org/abs/2509.15038). A
position whose key and value carry a large share of their neighbourhood's squared norm is kept longer.

API mirror of `kvpress/presses/cur_press.py`: the same fields and defaults (`compression_ratio` 0.0, `num_sinks` 4,
`leverage_type` "kv_product", `use_random_leverage` False, `use_local_approximation` True, `local_window_size` 16) and
the same `score()` contract, a `[B, Hkv, S]` tensor in the cache dtype where higher is kept longer. The score reads only
K and V: no queries, no hidden states, no attention weights.

The score, per row (include/kvpress_b200.h, kvp_cur_score; csrc/cur.cu):
    a_k = the squared norm of the key (of its projection by G with `use_random_leverage`), a_v of the value;
    with `use_local_approximation`, each is divided by its sum over its window of `local_window_size` positions
    (the last window may be short; an all-zero window is 0/0 = NaN, as in the reference);
    u = a_k | a_v | (a_k + a_v) / 2 | a_k a_v by `leverage_type`; score = u / sum of u over the row;
    the first `num_sinks` positions score 1.
The reference runs about a dozen cache-sized elementwise passes in the cache dtype. Here two sm_90a kernels read K and
V once, evaluate in fp32 and round once.

`use_random_leverage`: G = torch.randn(head_dim, 20, device=keys.device) / sqrt(20) is drawn in float32 on every
`score()` call, as the reference draws it (same generator, same shape, so the same draws under the same seed), and the
projection is done in fp32. The reference multiplies the cache by the float32 G directly, which torch refuses for
bf16 / fp16 caches, so there this option only ever worked on float32 caches.

`score()` reads `keys[..., a:b, :]` views in place (ChunkPress), with windows relative to the view. A
`local_window_size` above native.CUR_WINDOW_MAX (1024) scores through a float32 torch evaluation of the same definition
on the GPU; selection and compaction stay on the sm_90a kernels. A negative `num_sinks` is refused (in the reference it
would, through slicing, set everything but the last positions to 1).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import torch
from torch import nn

from kvpress_b200 import native
from kvpress_b200.presses.scorer_press import ScorerPress


def _cur_scores_fp32(keys: torch.Tensor, values: torch.Tensor, num_sinks: int, leverage_type: str, window: int,
                     G: Optional[torch.Tensor]) -> torch.Tensor:
    """The kernel's definition evaluated with float32 torch ops, rounded once to the cache dtype (windows above
    CUR_WINDOW_MAX). `window` 0: no local approximation."""
    S = keys.shape[2]

    def share(x: torch.Tensor) -> torch.Tensor:
        x = x.float()
        a = ((x @ G) if G is not None else x).square().sum(dim=-1)
        if window > 0:
            pad = (window - S % window) % window
            a = torch.nn.functional.pad(a, (0, pad)).unflatten(-1, (-1, window))
            a = (a / a.sum(dim=-1, keepdim=True)).flatten(-2)[..., :S]
        return a

    if leverage_type == "key":
        u = share(keys)
    elif leverage_type == "value":
        u = share(values)
    elif leverage_type == "kv_avg":
        u = (share(keys) + share(values)) / 2
    else:
        u = share(keys) * share(values)
    scores = u / u.sum(dim=-1, keepdim=True, dtype=torch.float64).float()
    scores[..., :num_sinks] = 1.0
    return scores.to(keys.dtype)


@dataclass
class CURPress(ScorerPress):
    """Keeps the positions with the largest approximate key / value leverage scores."""

    compression_ratio: float = 0.0
    num_sinks: int = 4
    leverage_type: str = "kv_product"
    use_random_leverage: bool = False
    use_local_approximation: bool = True
    local_window_size: int = 16

    needs_hidden_states = False

    def _arguments(self, keys: torch.Tensor):
        """(num_sinks, leverage_type, window, G) of one call; draws G."""
        if self.leverage_type not in native.CUR_LEVERAGE_TYPES:
            raise ValueError("Unknown leverage type: choose from 'kv_avg', 'key', 'value' or 'kv_product'")
        if self.num_sinks < 0:
            raise ValueError(f"num_sinks must not be negative, got {self.num_sinks}")
        window = 0
        if self.use_local_approximation:
            window = int(self.local_window_size)
            if window < 1:
                raise ValueError(f"local_window_size must be at least 1, got {self.local_window_size}")
        G = None
        if self.use_random_leverage:
            r = 20
            G = torch.randn(keys.shape[-1], r, device=keys.device) / math.sqrt(r)
        return self.num_sinks, self.leverage_type, window, G

    def score(self, module: nn.Module, hidden_states, keys: torch.Tensor, values, attentions, kwargs) -> torch.Tensor:
        num_sinks, leverage_type, window, G = self._arguments(keys)
        if window > native.CUR_WINDOW_MAX:
            return _cur_scores_fp32(keys, values, num_sinks, leverage_type, window, G)
        return native.cur_score(keys, values, num_sinks, leverage_type, window, G)

    def _fused_compress(self, module, hidden_states, keys, values, attentions, kwargs, n_kept):
        if self._score_is_overridden(CURPress):
            return None
        num_sinks, leverage_type, window, G = self._arguments(keys)
        if window > native.CUR_WINDOW_MAX:
            scores = _cur_scores_fp32(keys, values, num_sinks, leverage_type, window, G)
            return native.scores_compress(scores, keys, values, n_kept)[:2]
        k_out, v_out, _, _ = native.cur_compress(keys, values, num_sinks, leverage_type, window, G, n_kept)
        return k_out, v_out
