"""ObservedAttentionPress: importance = mean attention each key receives from the queries of the prompt (H2O,
https://arxiv.org/abs/2306.14048).

API mirror of `kvpress/presses/observed_attention_press.py`. The reference reduces the `[B, Hq, S, S]` weights that an
eager attention forward returns, which forces the whole model onto `attn_implementation="eager"` and materialises those
weights in every layer (48 GiB for one Llama-3.1-8B layer at 16k). Here the same score is recomputed from the queries
and the keys by two sm_90a tensor-core passes (csrc/observed_attention.cu): the exact softmax normaliser of every query
row, then the normalised column sums. Nothing of size S x S is formed, so the press runs under sdpa, flash and eager
alike, and `attentions` is accepted and ignored, as SnapKVPress does.

Host prologue (torch): the queries of the current forward, `q_proj` over the last n_q rows of `hidden_states` and RoPE
with the current `position_embeddings` (n_q = their length: S in prefill, the current step's rows under DecodingPress).
That query tensor is `[B, Hq, n_q, D]` in the cache dtype: 1 GiB for a Llama-3.1-8B layer at 128k.

The score is (1/G) sum over the G query heads of a kv head and over the query rows of the causal
softmax(module.scaling q.k), divided by S - s rounded to the cache dtype, as the reference divides by
`torch.arange(S, 0, -1)` in the attention dtype. In fp16 the counts of 65520 and above round to inf, so on prompts
longer than 65519 tokens the first positions score exactly 0 and are pruned first, as in the reference. The score is
evaluated in fp32 and rounded once to the cache dtype.

Head dims other than 64 / 128 and more than 8 query heads per kv head score through cuBLAS GEMMs
(wide_head_scores.py); selection and compaction stay on the sm_90a kernels.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch
from torch import nn

from kvpress_b200 import native, wide_head_scores
from kvpress_b200.presses.scorer_press import ScorerPress
from kvpress_b200.utils import apply_rope, get_prerope_query_states


@dataclass
class ObservedAttentionPress(ScorerPress):
    compression_ratio: float = 0.0

    def queries(self, module: nn.Module, hidden_states: torch.Tensor, keys: torch.Tensor, kwargs: dict) -> torch.Tensor:
        """RoPE'd queries of the current forward, [B, Hq, n_q, D] in the cache dtype."""
        S = keys.shape[2]
        cos, sin = kwargs["position_embeddings"]
        n_q = cos.shape[-2]
        if n_q > S:
            raise ValueError(f"{n_q} queries but only {S} cached positions: a press earlier in the chain already "
                             "pruned this layer's cache, so the causal mask cannot be placed")
        window = (module.sliding_window if hasattr(module, "sliding_window")
                  else getattr(module.config, "sliding_window", None))
        if window is not None and window < S:
            raise NotImplementedError(f"ObservedAttentionPress: the layer attends through a sliding window of {window} "
                                      f"< {S} positions; only the causal mask is implemented")
        q = get_prerope_query_states(module, hidden_states[:, -n_q:])
        return apply_rope(q, cos, sin).to(keys.dtype).contiguous()

    @staticmethod
    def _on_tensor_cores(keys: torch.Tensor, q: torch.Tensor) -> bool:
        return wide_head_scores.observed_attention_on_tensor_cores(keys.shape[-1], q.shape[1] // keys.shape[1])

    def score(self, module: nn.Module, hidden_states, keys: torch.Tensor, values, attentions, kwargs) -> torch.Tensor:
        q = self.queries(module, hidden_states, keys, kwargs)
        if not self._on_tensor_cores(keys, q):
            return wide_head_scores.observed_attention_scores(keys, q, module.scaling)
        return native.observed_attention_score(keys, q, module.scaling)

    def _fused_compress(self, module, hidden_states, keys, values, attentions, kwargs, n_kept):
        if self._score_is_overridden(ObservedAttentionPress):
            return None
        q = self.queries(module, hidden_states, keys, kwargs)
        if not self._on_tensor_cores(keys, q):
            scores = wide_head_scores.observed_attention_scores(keys, q, module.scaling)
            return native.scores_compress(scores, keys, values, n_kept)[:2]
        k_out, v_out, _, _ = native.observed_attention_compress(keys, values, q, module.scaling, n_kept)
        return k_out, v_out
