"""MergingPress: merge-on-evict around any ScorerPress. The wrapped press decides which rows survive, as it would alone;
before the others are dropped, every evicted value is folded into the kept row whose key is most cosine-similar,
weighted by that similarity and by the relative value norms. Keys are only gathered, so the press is safe under RoPE.

API mirror of `kvpress/presses/merging_press.py`: the same fields and defaults (`press` None, `similarity_threshold`
0.0, `merge_fraction` 1.0), the same `__post_init__` asserts, `post_init_from_model` and the `compression_ratio`
property that forwards to the wrapped press, and the public `merge(keys, values, indices)`.

The merge, per row (include/kvpress_b200.h, kvp_merging_compress; csrc/merging.cu): target(e) = the kept row of
largest cosine similarity with the evicted key e (ties to the lowest position); the merge proceeds where that
similarity is at least `similarity_threshold` and, with `merge_fraction` < 1, among the top `merge_fraction` of them
(torch.quantile's threshold, reproduced exactly); w = max(sim, 0) |v_e| / (|v_e| + |v_target| + 1e-6);
v_t <- (v_t + sum w v_e) / (1 + sum w). The reference forms the dense fp32 [B, Hkv, n_evict, n_kept] similarity tensor
(8.6 GB for a Llama-3.1-8B layer at 32k, 137 GB at 128k) and accumulates with scatter_add_, whose CUDA atomics make
two runs differ. Here an sm_90a tensor-core kernel keeps only a running argmax per evicted row, and the sums run in
ascending evicted position, the order of the reference's CPU scatter_add_: two calls are bitwise equal.

`compress` keeps the reference's uniform int(k_len * (1 - compression_ratio)) rows in every layer: it calls the wrapped
press's `score()` only, never its per-layer kept count (PyramidKVPress) or its fused compress path.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch
from torch import nn

from kvpress_b200 import native
from kvpress_b200.presses.base_press import BasePress
from kvpress_b200.presses.scorer_press import ScorerPress, kept_count


@dataclass
class MergingPress(BasePress):
    """Keeps the rows `press` keeps, after folding each evicted value into its most cosine-similar kept row."""

    press: ScorerPress = None  # type: ignore[assignment]
    similarity_threshold: float = 0.0
    merge_fraction: float = 1.0

    def __post_init__(self):
        assert isinstance(self.press, ScorerPress), (
            f"MergingPress requires a ScorerPress, got {type(self.press).__name__}"
        )
        assert 0.0 <= self.similarity_threshold <= 1.0
        assert 0.0 < self.merge_fraction <= 1.0, "merge_fraction must be in (0, 1]"

    def post_init_from_model(self, model):
        self.press.post_init_from_model(model)

    @property
    def compression_ratio(self) -> float:
        return self.press.compression_ratio

    @compression_ratio.setter
    def compression_ratio(self, value: float) -> None:
        self.press.compression_ratio = value

    def compress(self, module: nn.Module, hidden_states, keys: torch.Tensor, values: torch.Tensor, attentions,
                 kwargs: dict) -> tuple[torch.Tensor, torch.Tensor]:
        if self.press.compression_ratio == 0:
            return keys, values
        scores = self.press.score(module, hidden_states, keys, values, attentions, kwargs)
        n_kept = kept_count(keys.shape[2], self.press.compression_ratio)
        k_out, v_out, _, _, _ = native.merging_compress(scores, keys, values, self.similarity_threshold,
                                                        self.merge_fraction, n_kept)
        return k_out, v_out

    def merge(self, keys: torch.Tensor, values: torch.Tensor, indices: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        """The reference's merge: `indices` [B, Hkv, n_kept] are the kept positions in any order (scores.topk's). Returns
        the keys unchanged and full-shape values whose kept positions hold the merged rows."""
        S = keys.shape[2]
        n_kept = indices.shape[2]
        if n_kept == S or n_kept == 0:
            return keys, values
        kept = indices.sort(dim=-1).values
        if kept.numel() and (kept[..., 0].min() < 0 or kept[..., -1].max() >= S):
            raise ValueError(f"indices must lie in [0, {S})")
        if n_kept > 1 and (kept[..., 1:] == kept[..., :-1]).any():
            raise ValueError("indices must be distinct within every head")
        v_kept, _, _ = native.merging_merge(keys, values, kept, self.similarity_threshold, self.merge_fraction)
        out = values.clone()
        out.scatter_(2, kept.long().unsqueeze(-1).expand(-1, -1, -1, values.shape[3]), v_kept)
        return keys, out
