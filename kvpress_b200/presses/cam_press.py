"""CAMPress: Cache Merging (CaM, https://openreview.net/forum?id=LCTmppB165) while tokens are being generated.

API mirror of `kvpress/presses/cam_press.py`. It is DecodingPress plus two pieces of work:
  * every decoding step, in every layer, the attention of the current token over the whole cache is added into a
    running per-kv-head sum. The scan is the covariance-free ExpectedAttention kernel TOVAPress scores with (the group
    mean of softmax(q.k / sqrt(D)) of the RoPE'd last query); the sum is fp32 and lives in a capacity buffer that grows
    geometrically, so a step reallocates nothing;
  * every `compression_interval` steps, the base press's scores choose the `target_size` kept rows, and the values of
    up to k evicted positions (k: the steps since the last compaction) are merged, each with probability
    clamp(A[e] / window mean of A), into the `merge_budget` kept rows after them before K, V and the sum are compacted.
    That is one `kvp_cam_compress` call (include/kvpress_b200.h, which states the definition and its deviations from
    the reference: fp32 running sum, evicted set = complement of the kept set, fixed-order fp32 merge sums).
The merge draws come from `draw_uniforms` (torch.rand on the cache's device, so torch.manual_seed governs them).

The base press must be a ScorerPress. The reference also lists `CAMPress(AdaKVPress(SnapKVPress()))`, which fails there
at its first compaction (AdaKVPress has no `score`); that entry is not supported here and is rejected at construction.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch
import torch.nn as nn

from kvpress_b200 import native
from kvpress_b200.presses.decoding_press import DecodingPress
from kvpress_b200.presses.scorer_press import ScorerPress
from kvpress_b200.utils import extract_keys_and_values, last_query


def draw_uniforms(shape: tuple, device: torch.device) -> torch.Tensor:
    """The merge draws u [B, Hkv, n_merge] in [0, 1): candidate i of head j merges when u < p_i."""
    return torch.rand(shape, dtype=torch.float32, device=device)


class RunningAttention:
    """A layer's fp32 running attention sum [B, Hkv, length] inside a [B, Hkv, capacity] buffer, and the spare buffer
    a compaction writes the pruned sum into (the two are then swapped)."""

    def __init__(self, B: int, H: int, capacity: int, device: torch.device):
        self.buf = torch.zeros((B, H, capacity), dtype=torch.float32, device=device)
        self.spare = torch.empty_like(self.buf)
        self.length = 0

    def view(self) -> torch.Tensor:
        return self.buf[:, :, : self.length]

    def add(self, attn: torch.Tensor) -> None:
        """Adds the step's attention [B, Hkv, S]; the positions new since the last step start from 0."""
        B, H, S = attn.shape
        if self.buf.shape[:2] != (B, H) or S > self.buf.shape[2]:
            grown = RunningAttention(B, H, max(S, 2 * self.buf.shape[2]), attn.device)
            if self.buf.shape[:2] == (B, H):
                grown.buf[:, :, : self.length] = self.view()
                grown.length = self.length
            self.buf, self.spare = grown.buf, grown.spare
        self.buf[:, :, self.length: S].zero_()
        self.buf[:, :, :S] += attn
        self.length = S


@dataclass
class CAMPress(DecodingPress):
    """DecodingPress whose compaction merges some evicted values into the `merge_budget` kept rows after them.

    Parameters: base_press (a ScorerPress), compression_interval (decoding steps between compactions),
    target_size (rows kept by a compaction), hidden_states_buffer_size (hidden states buffered for the base press),
    merge_budget (kept rows after an evicted position that share its value)."""

    base_press: ScorerPress
    compression_interval: int = 512
    target_size: int = 2048
    hidden_states_buffer_size: int = 256
    merge_budget: int = 32

    def __post_init__(self):
        if not isinstance(self.base_press, ScorerPress):
            raise TypeError(f"CAMPress needs a ScorerPress base press (one with `score`), got "
                            f"{type(self.base_press).__name__}; AdaKVPress bases are not supported")
        super().__post_init__()
        assert self.merge_budget > 0, "merge_budget must be positive "
        self._running_attn_sum: dict[int, RunningAttention] = {}

    def _on_prefill(self, layer_idx: int) -> None:
        # a new sequence: no step, buffered hidden state or running sum of the last one survives
        self._running_attn_sum.pop(layer_idx, None)
        self.hidden_states_buffer[layer_idx] = []
        self.hidden_states_lens[layer_idx] = []
        self.layer_step_counts[layer_idx] = 0

    def _on_decoding_step(self, module: nn.Module, hidden_states: torch.Tensor, kwargs: dict) -> None:
        keys, values = extract_keys_and_values(kwargs["past_key_values"], module.layer_idx)
        attn = native.expected_attention_score(keys, values, last_query(module, hidden_states, kwargs), None, 0.0, 0,
                                               False)
        state = self._running_attn_sum.get(module.layer_idx)
        if state is None:
            state = self._running_attn_sum[module.layer_idx] = RunningAttention(*keys.shape[:3], keys.device)
        state.add(attn)

    def _should_compress(self, layer_idx: int, q_len: int, target: int, cache) -> bool:
        steps = self.layer_step_counts[layer_idx]
        return (steps >= self.compression_interval and cache.layers[layer_idx].keys.shape[2] > target) or \
            q_len >= target

    def compress(self, module: nn.Module, hidden_states, keys, values, attentions, kwargs: dict):
        layer_idx = module.layer_idx
        B, H, S, _ = keys.shape
        target = self.target_size
        if S <= target:
            return keys, values
        saved = self.base_press.compression_ratio
        self.base_press.compression_ratio = self._find_target_compression_ratio(S, target)
        try:
            scores = self.base_press.score(module, hidden_states, keys, values, None, kwargs)
        finally:
            self.base_press.compression_ratio = saved
        state = self._running_attn_sum[layer_idx]
        n_merge = min(self.layer_step_counts[layer_idx], S - target)
        u = draw_uniforms((B, H, n_merge), keys.device)
        keys, values, *_ = native.cam_compress(scores, keys, values, state.view(), state.spare[:, :, :target], n_merge,
                                               self.merge_budget, u, target)
        state.buf, state.spare, state.length = state.spare, state.buf, target
        return keys, values

    def reset(self):
        super().reset()
        self._running_attn_sum = {}
