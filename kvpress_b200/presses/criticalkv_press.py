"""CriticalKVPress / CriticalAdaKVPress: the wrapped press's scores, rescaled by how much each value moves the attention
output (https://arxiv.org/abs/2502.03805).

API mirror of `kvpress/presses/criticalkv_press.py:17-194`. Stage 1 keeps the `first_stage_ratio` share of the budget
by the wrapped press's score alone; stage 2 ranks the rest by (score + epsilon) * mean_g ||v_s Wo_h^T||_1 over the query
heads h of each kv head. The reference materialises V_h @ Wo_h, a [B, S, hidden] tensor per query head, to take its
row L1 norms; here the product never leaves the registers of the sm_90a kernel (csrc/criticalkv.cu). Head dims the
kernel does not instantiate score through cuBLAS GEMMs (wide_head_scores.py); selection stays on the sm_90a kernels.
"""
from __future__ import annotations

import logging
from dataclasses import dataclass

import torch
from torch import nn

from kvpress_b200 import native, wide_head_scores
from kvpress_b200.attention_patch import patch_attention_functions
from kvpress_b200.presses.base_press import BasePress
from kvpress_b200.presses.expected_attention_press import ExpectedAttentionPress
from kvpress_b200.presses.scorer_press import ScorerPress, kept_count

logger = logging.getLogger(__name__)


def _critical_scores(base: torch.Tensor, values: torch.Tensor, module: nn.Module, epsilon: float,
                     n_first: int) -> torch.Tensor:
    wo = module.o_proj.weight
    if not wide_head_scores.criticalkv_on_tensor_cores(values.shape[-1]):
        return wide_head_scores.criticalkv_scores(base, values, wo, epsilon, n_first)
    return native.criticalkv_score(base, values, wo, epsilon, n_first)


class CriticalKVPress(ScorerPress):
    """Two-stage selection over a ScorerPress: the n_first best positions by its score, then its score rescaled by the
    output-projected value norm."""

    def __init__(self, press: ScorerPress, epsilon: float = 1e-4, first_stage_ratio: float = 0.5):
        self.press = press
        self.epsilon = epsilon
        self.first_stage_ratio = first_stage_ratio
        assert isinstance(self.press, ScorerPress), "CriticalKVPress requires a ScorerPress as input"
        if isinstance(self.press, ExpectedAttentionPress) and self.press.use_vnorm:
            logger.warning("use_vnorm should be disabled for CriticalKVPress")

    def __repr__(self):
        return (f"CriticalKVPress(press={self.press!r}, epsilon={self.epsilon}, "
                f"first_stage_ratio={self.first_stage_ratio})")

    def post_init_from_model(self, model):
        self.press.post_init_from_model(model)

    @property  # type: ignore[misc]
    def compression_ratio(self):
        return self.press.compression_ratio

    @compression_ratio.setter
    def compression_ratio(self, value):
        self.press.compression_ratio = value

    @property  # type: ignore[misc]
    def needs_hidden_states(self):
        return getattr(self.press, "needs_hidden_states", True)

    def n_first(self, k_len: int) -> int:
        """Stage-1 budget, in the reference's float64 order (criticalkv_press.py:82)."""
        return int((1 - self.compression_ratio) * k_len * self.first_stage_ratio)

    def score(self, module: nn.Module, hidden_states, keys: torch.Tensor, values: torch.Tensor, attentions,
              kwargs) -> torch.Tensor:
        base = self.press.score(module, hidden_states, keys, values, attentions, kwargs)
        return _critical_scores(base, values, module, self.epsilon, self.n_first(keys.shape[2]))

    def _fused_compress(self, module, hidden_states, keys, values, attentions, kwargs, n_kept):
        n_first = self.n_first(keys.shape[2])
        if self._score_is_overridden(CriticalKVPress) or n_first > n_kept:
            return None
        if not wide_head_scores.criticalkv_on_tensor_cores(values.shape[-1]):
            return None  # score() runs the cuBLAS fallback; the generic selection follows
        base = self.press.score(module, hidden_states, keys, values, attentions, kwargs)
        k_out, v_out, _, _ = native.criticalkv_compress(base, keys, values, module.o_proj.weight, self.epsilon,
                                                        n_first, n_kept)
        return k_out, v_out


@dataclass
class CriticalAdaKVPress(BasePress):
    """CriticalKV with AdaKV's head-wise budgets (criticalkv_press.py:95-194): the cache keeps its shape and the pruned
    (batch, head, position) triples go to `module.masked_key_indices` for attention_patch.py."""

    press: ScorerPress = None
    alpha_safeguard: float = 0.20
    epsilon: float = 1e-4
    first_stage_ratio: float = 0.5

    def __post_init__(self):
        assert 0 <= self.alpha_safeguard <= 1, "alpha_safeguard should be in 0, 1]"
        assert isinstance(self.press, ScorerPress), "CriticalAdaKVPress requires a ScorerPress as input"
        if isinstance(self.press, ExpectedAttentionPress) and self.press.use_vnorm:
            logger.warning("use_vnorm should be disabled for CriticalAdaKVPress")
        patch_attention_functions()

    def post_init_from_model(self, model):
        self.press.post_init_from_model(model)

    @property
    def compression_ratio(self):
        return self.press.compression_ratio

    @compression_ratio.setter
    def compression_ratio(self, value):
        self.press.compression_ratio = value

    @staticmethod
    def _force_per_head(scores: torch.Tensor, budgets: list) -> None:
        """scores[:, h] gets finfo.max at its budgets[h] best positions (one selection per head, on its [B, 1, S] view)."""
        fmax = torch.finfo(scores.dtype).max
        for h, budget in enumerate(budgets):
            if budget > 0:
                view = scores[:, h:h + 1, :]
                view.scatter_(-1, native.scores_select(view, min(budget, scores.shape[2])).long(), fmax)

    def compress(self, module: nn.Module, hidden_states, keys: torch.Tensor, values: torch.Tensor, attentions,
                 kwargs: dict) -> tuple[torch.Tensor, torch.Tensor]:
        if self.compression_ratio == 0:
            return keys, values
        assert module.config._attn_implementation != "eager", "eager mode not supported"
        scores = self.press.score(module, hidden_states, keys, values, attentions, kwargs)
        B, H, S = scores.shape
        fmax = torch.finfo(scores.dtype).max

        # at least alpha * n_kept positions per head (:148-152)
        n_kept = kept_count(S, self.compression_ratio)
        n_safe = int(n_kept * self.alpha_safeguard)
        if n_safe > 0:
            scores = scores.scatter(-1, native.scores_select(scores, n_safe).long(), fmax)

        # head budgets: heads of the n_kept * H best positions of the head-flattened rows, summed over the batch
        # (:158-164); one host read of the budgets and their stage-1 shares (:167)
        flat = native.scores_select(scores.reshape(B, 1, H * S), n_kept * H).long()
        head_budgets = torch.bincount((flat // S).flatten(), minlength=H)
        first = (head_budgets * self.first_stage_ratio).to(torch.int64)
        budgets, budgets_1st = torch.stack([head_budgets, first]).tolist()

        # stage 1 (:167-171), stage 2 (:174-179)
        self._force_per_head(scores, budgets_1st)
        scores = _critical_scores(scores, values, module, self.epsilon, 0)
        self._force_per_head(scores, budgets)

        # bottom-k across heads (:186-193)
        n_pruned = H * (S - n_kept)
        flat = native.scores_select((-scores).reshape(B, 1, H * S), n_pruned).reshape(-1).long()
        batch = torch.arange(B, device=flat.device).repeat_interleave(n_pruned)
        module.masked_key_indices = (batch, flat // S, flat % S)
        return keys, values
