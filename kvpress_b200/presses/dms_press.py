"""DMSPress: evict every position whose score falls below a threshold (https://arxiv.org/abs/2506.05345, dense prefill).

API mirror of `kvpress/presses/dms_press.py`. It wraps a ScorerPress, keeps a per-layer buffer of the scores of the
positions that have not been judged yet, protects the `sliding_window_size` most recent ones, and marks every older
position scoring below `threshold` in `module.masked_key_indices`, which attention_patch.py turns into keys no query
attends to. The cache keeps its shape; the achieved ratio depends on the input (`compression_ratio` is read-only, the
mean of the per-layer `compression_ratios`). With `decoding=True` the pipeline keeps the press live while generating.

Differences from the reference: the phase comes from hook_is_prefilling (no `.item()`); the positions are found by
`kvp_threshold_evict` (csrc/kvzap.cu), exact and in `torch.where` order, with one host read of their count per hook
call; the absolute position of a buffered score is taken from the cache length instead of `cache_position`, the same
number when nothing else shortens the cache.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Optional

import torch
from torch import nn

from kvpress_b200 import native
from kvpress_b200.attention_patch import patch_attention_functions
from kvpress_b200.presses.base_press import BasePress, hook_is_prefilling
from kvpress_b200.presses.scorer_press import ScorerPress
from kvpress_b200.utils import extract_keys_and_values


@dataclass
class DMSPress(BasePress):
    """Masks the positions older than the sliding window whose `press` score is below `threshold`."""

    press: ScorerPress
    threshold: Optional[float] = None
    sliding_window_size: int = 128
    decoding: bool = False
    scores_buffer: dict = field(default_factory=dict, init=False, repr=False)
    compression_ratios: dict = field(default_factory=dict, init=False, repr=False)

    def __post_init__(self):
        assert isinstance(self.press, ScorerPress), "DMSPress requires a ScorerPress as input"
        patch_attention_functions()

    def post_init_from_model(self, model):
        self.press.post_init_from_model(model)

    @property
    def compression_ratio(self):
        """Mean over the layers of the masked share of the cache (known after a forward pass)."""
        assert len(self.compression_ratios) > 0, "Forward pass must be run to compute the compression ratio"
        return sum(self.compression_ratios.values()) / len(self.compression_ratios)

    @compression_ratio.setter
    def compression_ratio(self, value):
        raise AttributeError(f"compression ratio cannot be set for {type(self).__name__}")

    def forward_hook(self, module: nn.Module, input: list, kwargs: dict, output: list):
        hidden_states = kwargs["hidden_states"]
        q_len = hidden_states.shape[1]
        layer_idx: int = module.layer_idx
        prefilling = hook_is_prefilling(module, kwargs)
        if prefilling and layer_idx == 0:
            self.scores_buffer.clear()
            self.compression_ratios.clear()
        if not prefilling and not self.decoding:
            return output
        if self.threshold is None:
            raise ValueError("DMSPress needs a threshold: set DMSPress(press, threshold=...)")

        keys, values = extract_keys_and_values(kwargs["past_key_values"], layer_idx)
        scores = self.press.score(module, hidden_states, keys[:, :, -q_len:], values[:, :, -q_len:], None, kwargs)
        buffer = scores if prefilling else torch.cat([self.scores_buffer[layer_idx], scores], dim=-1)

        if buffer.shape[-1] > self.sliding_window_size:
            n_evict = buffer.shape[-1] - self.sliding_window_size
            # buffer position 0 is cache position cache_len - buffer length
            shift = keys.shape[2] - buffer.shape[-1]
            new = native.threshold_evict(buffer, n_evict, self.threshold, shift)
            buffer = buffer[..., n_evict:]
            if new[0].numel() > 0:
                old = getattr(module, "masked_key_indices", None)
                module.masked_key_indices = new if old is None else [torch.cat([i, n]) for i, n in zip(old, new)]
        self.scores_buffer[layer_idx] = buffer

        masked = getattr(module, "masked_key_indices", None)
        if masked is not None:
            B, H, S, _ = keys.shape
            self.compression_ratios[layer_idx] = len(masked[0]) / (B * H * S)
        else:
            self.compression_ratios[layer_idx] = 0
        return output
