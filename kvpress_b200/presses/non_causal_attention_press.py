"""NonCausalAttnPress: importance = non-causal, chunked attention each key receives from the queries of its chunk, times
||v||, pooled and z-normalised; the attention half of Compactor (Chari & Van Durme, 2025,
https://arxiv.org/abs/2507.08143).

API mirror of `kvpress/presses/non_causal_attention_press.py`: the same fields (`compression_ratio`, `chunk_size` = 256),
the same prefill-only assert and the same `score()` contract, a `[B, Hkv, S]` tensor where higher is kept longer. The
reference forms `[B, Hq, S/cs, cs, cs]` logits in the cache dtype, an fp32 copy and the fp32 softmax (10 GiB for one
Llama-3.1-8B layer at 128k with cs = 256); here one sm_90a tensor-core kernel (csrc/non_causal_attention.cu) computes
every chunk's exact softmax normalisers and column sums in shared memory and registers, and nothing of size cs x cs
reaches global memory.

Host prologue (torch): `q_proj` over `hidden_states` and RoPE with the last S rows of `position_embeddings`, as the
reference does. That query tensor is `[B, Hq, S, D]` in the cache dtype: 1 GiB for a Llama-3.1-8B layer at 128k.

The score, per kv head j and position s with G = Hq / Hkv (include/kvpress_b200.h, kvp_non_causal_attention_score):
    A[h, s]  = sum over the queries i of s's chunk of softmax over the chunk's keys of q_i . k (unscaled logits)
    x[j, s]  = mean_g A[j G + g, s] * ||v[j, s]||,   pooled = avg_pool1d(x, 3, padding 1),
    score    = (pooled - mean) / std.clamp_min(1e-6), mean and unbiased std over ALL B * Hkv * S entries.
The padded last chunk follows the reference's quirk: the padded keys are not masked out (logit -1e-9, i.e. 0) and each
padded query row adds 1/cs to every valid key of that chunk. Because the z-score is global, the rows of a batch are
coupled, and a single entry (B * Hkv * S = 1) scores NaN, as in the reference.

The reference rounds the logits to the cache dtype before its fp32 softmax; with unscaled logits of magnitude 10-100 that
moves probabilities by tens of percent, so on real models parity with the reference is loose by construction. Here the
formula is evaluated in fp32 from the 16-bit inputs and rounded once to the cache dtype (the reference returns fp32);
selection keeps the n_kept largest of those rounded scores, ties to the lowest positions.

`score()` takes `keys[..., a:b, :]` views with the matching slices of `hidden_states` and `position_embeddings`
(CompactorPress scores segments that way); such views are read in place through the kernel's TMA map.

Head dims other than 64 / 128, more than 8 query heads per kv head and chunk sizes other than 128 / 256 score through
torch GEMMs on the GPU (wide_head_scores.py); selection and compaction stay on the sm_90a kernels.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch
from torch import nn

from kvpress_b200 import native, wide_head_scores
from kvpress_b200.presses.scorer_press import ScorerPress
from kvpress_b200.utils import apply_rope, get_prerope_query_states


@dataclass
class NonCausalAttnPress(ScorerPress):
    compression_ratio: float = 0.0
    chunk_size: int = 256

    def queries(self, module: nn.Module, hidden_states: torch.Tensor, keys: torch.Tensor, kwargs: dict) -> torch.Tensor:
        """RoPE'd queries of every cached position, [B, Hq, S, D] in the cache dtype."""
        assert keys.shape[-2] == hidden_states.shape[-2], "NonCausalAttnPress only supports prefill"
        assert self.chunk_size > 0, "chunk_size must be positive"
        cos, sin = kwargs["position_embeddings"]
        q = get_prerope_query_states(module, hidden_states)
        q_len = q.shape[-2]
        return apply_rope(q, cos[:, -q_len:], sin[:, -q_len:]).to(keys.dtype).contiguous()

    def _on_tensor_cores(self, keys: torch.Tensor, q: torch.Tensor) -> bool:
        return wide_head_scores.non_causal_attention_on_tensor_cores(keys.shape[-1], q.shape[1] // keys.shape[1],
                                                                     self.chunk_size)

    def score(self, module: nn.Module, hidden_states, keys: torch.Tensor, values, attentions, kwargs) -> torch.Tensor:
        q = self.queries(module, hidden_states, keys, kwargs)
        if not self._on_tensor_cores(keys, q):
            return wide_head_scores.non_causal_attention_scores(keys, values, q, self.chunk_size)
        return native.non_causal_attention_score(keys, values, q, self.chunk_size)

    def _fused_compress(self, module, hidden_states, keys, values, attentions, kwargs, n_kept):
        if self._score_is_overridden(NonCausalAttnPress):
            return None
        q = self.queries(module, hidden_states, keys, kwargs)
        if not self._on_tensor_cores(keys, q):
            scores = wide_head_scores.non_causal_attention_scores(keys, values, q, self.chunk_size)
            return native.scores_compress(scores, keys, values, n_kept)[:2]
        k_out, v_out, _, _ = native.non_causal_attention_compress(keys, values, q, self.chunk_size, n_kept)
        return k_out, v_out
