"""DecodingPress: periodic compaction of the cache while tokens are being generated.

API mirror of `kvpress/presses/decoding_press.py:22-239`: every
`compression_interval` forward calls of a layer (or when a multi-token call is at least
`target_size` long) the layer's cache is compacted to exactly `target_size` positions with the
wrapped scorer press, whose `compression_ratio` is set for the duration of that call.

Differences that do not change results:
  * decoding is detected from Python ints (no `.item()` sync per layer per token);
  * hidden states are only buffered (and cloned) when the wrapped press reads them
    (`needs_hidden_states`); Knorm / StreamingLLM never do, which removes a [B,1,hidden] clone per
    layer per generated token. A press that reads only the LENGTH of the buffered hidden states
    (`needs_hidden_states_len`: ExpectedAttentionStatsPress derives the future RoPE positions from it)
    gets a zero-copy stride-0 view of the length the reference's buffer would have;
  * the compaction itself is the fused sm_90a path of the wrapped press.
"""
from __future__ import annotations

import logging
from collections import defaultdict
from contextlib import contextmanager
from dataclasses import dataclass

import torch
import torch.nn as nn
from transformers import PreTrainedModel

from kvpress_b200.presses.base_press import BasePress, hook_is_prefilling, write_back
from kvpress_b200.presses.scorer_press import ScorerPress, kept_count
from kvpress_b200.utils import extract_keys_and_values

logger = logging.getLogger(__name__)


_RATIO_CACHE: dict = {}


def find_target_compression_ratio(k_len: int, target: int, max_iterations: int = 20) -> float:
    """Ratio r with int(k_len * (1 - r)) == target, found by the reference's bisection
    (decoding_press.py:194-236); 0.0 when the cache is already at or below the target. A decoding run asks for
    the same two or three (k_len, target) pairs thousands of times (once per layer per compaction): memoised."""
    key = (k_len, target, max_iterations)
    hit = _RATIO_CACHE.get(key)
    if hit is None:
        if len(_RATIO_CACHE) > 4096:
            _RATIO_CACHE.clear()
        hit = _RATIO_CACHE[key] = _find_target_compression_ratio(k_len, target, max_iterations)
    return hit


def _find_target_compression_ratio(k_len: int, target: int, max_iterations: int = 20) -> float:
    if k_len <= target:
        return 0.0
    ratio = 1.0 - target / k_len
    low, high = 0.0, 1.0
    for _ in range(max_iterations):
        kept = kept_count(k_len, ratio)
        if kept == target:
            break
        if kept > target:  # compress more
            low = ratio
            ratio = (ratio + high) / 2
        else:  # compress less
            high = ratio
            ratio = (low + ratio) / 2
    if kept_count(k_len, ratio) != target:
        logger.warning(f"Binary search failed: q_len={k_len}, target={target}, "
                       f"got={kept_count(k_len, ratio)}, ratio={ratio}")
    return ratio


@dataclass
class DecodingPress(BasePress):
    """Applies `base_press` every `compression_interval` decoding steps down to `target_size` positions."""

    base_press: ScorerPress
    compression_interval: int = 512
    target_size: int = 2048
    hidden_states_buffer_size: int = 256

    def __post_init__(self):
        assert isinstance(self.base_press, ScorerPress), "DecodingPress requires a ScorerPress as input"
        assert self.compression_interval > 0, "compression_interval must be greater than 0"
        assert self.target_size > 0, "target_size must be greater than 0"
        self.hidden_states_buffer = defaultdict(list)  # layer_idx -> list of [B, q, hidden]
        self.hidden_states_lens = defaultdict(list)    # layer_idx -> q_len of every buffered chunk (length-only presses)
        self.layer_step_counts = defaultdict(int)
        if self.base_press.compression_ratio:
            logger.warning(
                f"compression_ratio is set for base press ({self.base_press.compression_ratio}). "
                f"This will be overridden by the decoding press."
            )

    def post_init_from_model(self, model):
        self.base_press.post_init_from_model(model)

    def _resolve_target_size(self, kwargs: dict) -> int:
        return self.target_size

    def _find_target_compression_ratio(self, q_len: int, target_tokens: int) -> float:
        return find_target_compression_ratio(q_len, target_tokens)

    def compress(self, module: nn.Module, hidden_states, keys, values, attentions, kwargs: dict):
        """Delegate to the base press with the ratio that yields exactly `target_size` positions."""
        k_len = keys.shape[2]
        target = self._resolve_target_size(kwargs)
        ratio = self._find_target_compression_ratio(k_len, target)
        logger.debug(f"Compressing {k_len} to {target} with ratio {ratio}")
        saved = self.base_press.compression_ratio
        self.base_press.compression_ratio = ratio
        try:
            return self.base_press.compress(module, hidden_states, keys, values, attentions, kwargs)
        finally:
            self.base_press.compression_ratio = saved

    def forward_hook(self, module: nn.Module, input: list[torch.Tensor], kwargs: dict, output: list):
        hidden_states = kwargs["hidden_states"]
        cache = kwargs["past_key_values"]
        q_len = hidden_states.shape[1]
        layer_idx = module.layer_idx
        if hook_is_prefilling(module, kwargs):
            self._on_prefill(layer_idx)
            return output  # prefill is some other press's business

        buffering = self.hidden_states_buffer_size > 0 and getattr(self.base_press, "needs_hidden_states", True)
        length_only = (not buffering and self.hidden_states_buffer_size > 0
                       and getattr(self.base_press, "needs_hidden_states_len", False))
        if buffering:
            self.hidden_states_buffer[layer_idx].append(hidden_states.detach().clone())
        elif length_only:
            self.hidden_states_lens[layer_idx].append(q_len)
        self.layer_step_counts[layer_idx] += 1
        self._on_decoding_step(module, hidden_states, kwargs)

        target = self._resolve_target_size(kwargs)
        if self._should_compress(layer_idx, q_len, target, cache):
            logger.debug(f"Applying decoding compression at layer {layer_idx}: "
                         f"step {self.layer_step_counts[layer_idx]} / interval {self.compression_interval}")
            keys, values = extract_keys_and_values(cache, layer_idx)
            attentions = output[1] if len(output) > 1 and output[1] is not None else None
            if buffering:
                buffered = torch.cat(self.hidden_states_buffer[layer_idx], dim=1)
            elif length_only:  # same shape as the reference's concatenated buffer, no data
                total = sum(self.hidden_states_lens[layer_idx])
                buffered = hidden_states[:, :1].expand(-1, total, -1)
            else:
                buffered = hidden_states
            keys, values = self.compress(module, buffered, keys, values, attentions, kwargs)
            logger.debug(f"Applied decoding compression: keys.shape: {keys.shape}, values.shape: {values.shape}")
            write_back(cache, layer_idx, keys, values)
            self.layer_step_counts[layer_idx] = 0
            self.hidden_states_buffer[layer_idx] = []  # buffer and cache must stay aligned
            self.hidden_states_lens[layer_idx] = []

        if buffering:
            self.hidden_states_buffer[layer_idx] = self.hidden_states_buffer[layer_idx][-self.hidden_states_buffer_size:]
        elif length_only:
            self.hidden_states_lens[layer_idx] = self.hidden_states_lens[layer_idx][-self.hidden_states_buffer_size:]
        return output

    def _on_prefill(self, layer_idx: int) -> None:
        """Called by the hook on a prefill forward of a layer (DecodingPress keeps its state)."""

    def _on_decoding_step(self, module: nn.Module, hidden_states: torch.Tensor, kwargs: dict) -> None:
        """Called by the hook on every decoding forward of a layer, after the step is counted, before any compaction."""

    def _should_compress(self, layer_idx: int, q_len: int, target: int, cache) -> bool:
        return self.layer_step_counts[layer_idx] >= self.compression_interval or q_len >= target

    def reset(self):
        self.hidden_states_buffer = defaultdict(list)
        self.hidden_states_lens = defaultdict(list)
        self.layer_step_counts = defaultdict(int)

    @contextmanager
    def __call__(self, model: PreTrainedModel):
        try:
            with super().__call__(model):
                yield
        finally:
            self.reset()
