"""ThinKPress: channel-wise key compression (https://arxiv.org/abs/2407.21018). It zeroes the key CHANNELS that matter
least to the last `window_size` queries and removes no position, so it composes with every sequence press, e.g.
`ComposedPress([SnapKVPress(0.5), ThinKPress(0.5)])`.

API mirror of `kvpress/presses/think_press.py`: the same fields and defaults (`key_channel_compression_ratio` 0.0,
`window_size` 32), the same window queries (the last window_size positions, all of them for a shorter prompt, RoPE'd),
`compression_ratio` = key_channel_compression_ratio / 2 with a setter that raises. Per kv head, channel c scores
qn(c) kn(c): its mean square over the window queries of the head's query group times its mean square over the cached
positions; the int(head_dim * ratio) lowest-scoring channels are set to +0 at every position.

The reference squares the whole cache into a bf16 temporary, ranks bf16-rounded scores and scatters zeros. Here one
sm_90a kernel reads K once and ranks fp32 scores (ties: the higher channel is pruned; NaN last), and a second one
zeroes the pruned channels in place (include/kvpress_b200.h, kvp_think_prune; csrc/think.cu). The keys and values
returned are the tensors the press was given.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch
from torch import nn

from kvpress_b200 import native
from kvpress_b200.presses.base_press import BasePress
from kvpress_b200.utils import apply_rope, get_prerope_query_states


@dataclass
class ThinKPress(BasePress):
    """Zeroes the key channels least used by the last window_size queries."""

    key_channel_compression_ratio: float = 0.0
    window_size: int = 32

    def __post_init__(self):
        self._n_pruned(0)

    def _n_pruned(self, head_dim: int) -> int:
        r = self.key_channel_compression_ratio
        if not 0.0 <= r <= 1.0:
            raise ValueError(f"key_channel_compression_ratio must be in [0, 1], got {r}")
        return int(head_dim * r)

    def compute_window_queries(self, module: nn.Module, hidden_states: torch.Tensor, position_embeddings):
        """RoPE'd queries of the last window_size positions (all of them for a shorter prompt), [B, Hq, w, D]."""
        w = self.window_size
        q = get_prerope_query_states(module, hidden_states[:, -w:])
        cos, sin = position_embeddings
        return apply_rope(q, cos[:, -w:], sin[:, -w:])

    def compress(self, module: nn.Module, hidden_states, keys: torch.Tensor, values: torch.Tensor, attentions,
                 kwargs: dict) -> tuple[torch.Tensor, torch.Tensor]:
        n_pruned = self._n_pruned(keys.shape[-1])
        if self.key_channel_compression_ratio == 0:
            return keys, values
        q = self.compute_window_queries(module, kwargs["hidden_states"], kwargs["position_embeddings"])
        native.think_prune(keys, q.to(keys.dtype), n_pruned)
        return keys, values

    @property
    def compression_ratio(self):
        return self.key_channel_compression_ratio / 2

    @compression_ratio.setter
    def compression_ratio(self, value):
        raise AttributeError(f"compression ratio cannot be set for {type(self).__name__}")
