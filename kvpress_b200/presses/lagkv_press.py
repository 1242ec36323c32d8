"""LagKVPress: lag-relative KV cache compression (https://arxiv.org/abs/2504.04704). The cache after the sinks is cut into
partitions of `lag_size` positions; each partition's keys and values are scaled by the per-channel min / max of the
NEXT partition, and the spread of a position's scaled channels says how much it stands out.

API mirror of `kvpress/presses/lagkv_press.py`: the same fields and defaults (`compression_ratio` 0.0, `n_sink` 4,
`lag_size` 128, `cross_scoring` False) and the same `score()` contract, a `[B, Hkv, S]` tensor in the cache dtype where
higher is kept longer. The score reads only K and V: no queries, no hidden states, no attention weights.

The score, per row (include/kvpress_b200.h, kvp_lagkv_score; csrc/lagkv.cu):
    short cache (S < n_sink + 2 lag_size): 1 on the sinks, then the ramp (s - n_sink) / (S - n_sink);
    otherwise, per scored partition c (every partition but the last, which is its successor's reference):
        x = (k - lo) / (hi - lo) per channel, lo / hi the min / max of partition c + 1,
        sigma = unbiased std of x over the channels, a = softmax of sigma over the partition, for K and for V,
        c = (a_k + a_v) / 2, and the score is c (cross_scoring) or its rank within the partition / lag_size;
    the sinks, the last partition and the remainder score 1.
The reference writes and reads back cache-sized temporaries in the cache dtype and runs the whole chain in it (a bf16
combined score takes about ten distinct values per 128-row partition, so its ranks are mostly the tie order of its
argsort). Here one sm_90a kernel reads K and V about once, evaluates in fp32 and rounds once; rank ties go to the
earlier position. A constant channel of a reference partition (a zeroed channel, or lag_size 1) makes the partition it
scores NaN: its ranks are in position order and its cross scores NaN, as in the reference.

`score()` reads `keys[..., a:b, :]` views in place (ChunkPress). lag_size above native.LAG_MAX (1024) scores through a
float32 torch evaluation of the same definition on the GPU; selection and compaction stay on the sm_90a kernels.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch
from torch import nn

from kvpress_b200 import native
from kvpress_b200.presses.scorer_press import ScorerPress


def _lagkv_scores_fp32(keys: torch.Tensor, values: torch.Tensor, n_sink: int, lag_size: int,
                       cross_scoring: bool) -> torch.Tensor:
    """The kernel's definition evaluated with float32 torch ops, rounded once to the cache dtype (lag_size > LAG_MAX)."""
    B, H, S, D = keys.shape
    out = torch.ones((B, H, S), dtype=torch.float32, device=keys.device)
    if S < n_sink + 2 * lag_size:
        if S > n_sink:
            out[..., n_sink:] = torch.arange(S - n_sink, device=keys.device, dtype=torch.float32) / float(S - n_sink)
        return out.to(keys.dtype)
    P = (S - n_sink) // lag_size
    end = n_sink + P * lag_size

    def softmax_of_sigma(x: torch.Tensor) -> torch.Tensor:
        t = x[:, :, n_sink:end].float().reshape(B, H, P, lag_size, D)
        lo = t[:, :, 1:].amin(dim=-2, keepdim=True)
        hi = t[:, :, 1:].amax(dim=-2, keepdim=True)
        return ((t[:, :, :-1] - lo) / (hi - lo)).std(dim=-1).softmax(dim=-1)

    c = (softmax_of_sigma(keys) + softmax_of_sigma(values)) / 2
    if not cross_scoring:
        # a stable sort puts NaN last and keeps equal values in position order: the rank of the definition
        order = torch.sort(c, dim=-1, stable=True).indices
        c = order.argsort(dim=-1).to(torch.float32) / float(lag_size)
    out[..., n_sink:end - lag_size] = c.reshape(B, H, -1)
    return out.to(keys.dtype)


@dataclass
class LagKVPress(ScorerPress):
    """Keeps the positions whose keys and values stand out most against the next partition's range."""

    compression_ratio: float = 0.0
    n_sink: int = 4
    lag_size: int = 128
    cross_scoring: bool = False

    needs_hidden_states = False

    def score(self, module: nn.Module, hidden_states, keys: torch.Tensor, values, attentions, kwargs) -> torch.Tensor:
        if self.lag_size > native.LAG_MAX:
            return _lagkv_scores_fp32(keys, values, self.n_sink, self.lag_size, self.cross_scoring)
        return native.lagkv_score(keys, values, self.n_sink, self.lag_size, self.cross_scoring)

    def _fused_compress(self, module, hidden_states, keys, values, attentions, kwargs, n_kept):
        if self._score_is_overridden(LagKVPress):
            return None
        if self.lag_size > native.LAG_MAX:
            scores = _lagkv_scores_fp32(keys, values, self.n_sink, self.lag_size, self.cross_scoring)
            return native.scores_compress(scores, keys, values, n_kept)[:2]
        k_out, v_out, _, _ = native.lagkv_compress(keys, values, self.n_sink, self.lag_size, self.cross_scoring, n_kept)
        return k_out, v_out
