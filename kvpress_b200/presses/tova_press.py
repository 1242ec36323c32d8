"""TOVAPress: importance = attention the LAST token pays to each earlier key, averaged over all heads
(https://arxiv.org/abs/2401.06104).

API mirror of `kvpress/presses/tova_press.py:16-61`. The per-head softmax(q_last . k / sqrt(d)) over
all S keys is exactly the covariance-free ExpectedAttention scan with mu := the RoPE'd query of the last position,
no sinks, no value norms — so the cache pass is `kvp_expected_attention_score` (one streaming read of K, fp32
softmax, mean over the query heads of each kv head). The remaining ops are `[B, Hkv, S]`-sized: mean over kv heads
(all heads share one score row, as in the reference), and the last position is forced with max + 1 (computed on the
device, no host sync). `attentions` (eager weights) is accepted and ignored, like in SnapKVPress.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch
from torch import nn

from kvpress_b200 import native
from kvpress_b200.presses.scorer_press import ScorerPress
from kvpress_b200.utils import last_query


@dataclass
class TOVAPress(ScorerPress):
    compression_ratio: float = 0.0

    def last_query(self, module: nn.Module, hidden_states: torch.Tensor, kwargs: dict) -> torch.Tensor:
        """RoPE'd query of the last position, [B, Hq, D]."""
        return last_query(module, hidden_states, kwargs)

    def score(self, module: nn.Module, hidden_states, keys: torch.Tensor, values, attentions, kwargs) -> torch.Tensor:
        H = keys.shape[1]
        q_last = self.last_query(module, hidden_states, kwargs)
        per_kv_head = native.expected_attention_score(keys, values, q_last, None, 0.0, 0, False)   # [B, Hkv, S]
        shared = per_kv_head.float().mean(dim=1, keepdim=True).to(keys.dtype)
        scores = shared.expand(-1, H, -1).clone()
        scores[..., -1] = scores[..., :-1].amax() + 1        # the last token is always kept
        return scores
