"""FinchPress: SnapKV with the window set by the prompt (FINCH, https://direct.mit.edu/tacl/article/doi/10.1162/tacl_a_00716).

API mirror of `kvpress/presses/finch_press.py`. The prompt is `context + delimiter + question`: a forward hook on
`embed_tokens` finds the delimiter, drops its embedding and sets `window_size` to the question's length. Every
question token is a window query; each context key scores the attention the window pays to it, every window row
weighted by its position count c_i = S - w + i (`normalize_scores`), averaged over the G w rows of its kv head. The
window is always kept. With `chunk_length`, each chunk of positions keeps its own best max(1, int(len (1 - r))), and
with `rerotate_keys` the kept keys are re-rotated to their new, contiguous positions.

Everything that touches the cache runs in sm_90a kernels (include/kvpress_b200.h, kvp_finch_compress; csrc/finch.cu):
the window attention is recomputed from Q and K through TMA and wgmma without forming repeat_kv(K), the
[B, Hq, w, S] logits, their mask or an fp32 softmax copy, and the selection, gather and re-rotation follow in the
same call. The weights c_i are exact integers in fp32; the reference rounds them to the cache dtype (fp16 gives inf
from 65520 on). Shapes the kernels do not instantiate (head_dim other than 64 / 128, more than 8 query heads per kv
head) are scored with blocked cuBLAS GEMMs (finch_wide_head.finch_scores) and selected on the sm_90a kernels.

`attentions` (eager attention weights) is accepted for signature compatibility and ignored, as in SnapKVPress.
"""
from __future__ import annotations

from contextlib import contextmanager
from dataclasses import dataclass, field
from typing import Optional

import torch
from torch import nn

from kvpress_b200 import finch_wide_head, native
from kvpress_b200.presses.base_press import BasePress
from kvpress_b200.utils import apply_rope, get_prerope_query_states


@dataclass
class FinchPress(BasePress):
    compression_ratio: float = 0.0
    chunk_length: Optional[int] = None
    normalize_scores: bool = True
    rerotate_keys: bool = True
    delimiter_token: str = field(default=None, init=False)
    delimiter_token_id: int = field(default=None, init=False)
    window_size: int = field(default=None, init=False)

    def window_queries(self, module: nn.Module, hidden_states: torch.Tensor, kwargs: dict) -> torch.Tensor:
        """RoPE'd queries of the last `window_size` positions (the question), [B, Hq, w, D]."""
        w = self.window_size
        assert w is not None, "window_size must be provided"
        q = get_prerope_query_states(module, hidden_states[:, -w:])
        cos, sin = kwargs["position_embeddings"]
        return apply_rope(q, cos[:, -w:], sin[:, -w:])

    def _check_window(self, keys: torch.Tensor) -> None:
        if not 1 <= self.window_size < keys.shape[2]:
            raise ValueError(f"window_size {self.window_size} must be in [1, {keys.shape[2]}) for {keys.shape[2]} "
                             "cached positions")

    def score(self, module: nn.Module, hidden_states, keys: torch.Tensor, values, attentions, kwargs) -> torch.Tensor:
        """[B, Hkv, S] scores in the cache dtype, the window positions holding the reference's max + 1."""
        self._check_window(keys)
        q = self.window_queries(module, hidden_states, kwargs).to(keys.dtype)
        if not finch_wide_head.finch_on_tensor_cores(keys.shape[-1], q.shape[1] // keys.shape[1]):
            return finch_wide_head.finch_scores(keys, q, self.window_size, self.normalize_scores)
        return native.finch_score(keys, q, self.window_size, self.normalize_scores)

    def compress(self, module: nn.Module, hidden_states, keys: torch.Tensor, values: torch.Tensor, attentions,
                 kwargs: dict) -> tuple[torch.Tensor, torch.Tensor]:
        if self.compression_ratio == 0:
            return keys, values
        assert self.window_size is not None, "window_size must be provided"
        if self.chunk_length is not None:
            assert self.chunk_length > self.window_size / (1 - self.compression_ratio)
        self._check_window(keys)
        inv_freq = module.rotary_emb.inv_freq if self.rerotate_keys else None
        q = self.window_queries(module, hidden_states, kwargs).to(keys.dtype)
        if not finch_wide_head.finch_on_tensor_cores(keys.shape[-1], q.shape[1] // keys.shape[1]):
            scores = finch_wide_head.finch_scores(keys, q, self.window_size, self.normalize_scores)
            # the window is forced, as the kernels force it: max + 1 may round back to max in the cache dtype
            scores[..., -self.window_size:] = float("inf")
            if self.chunk_length is None:
                n_kept = int(keys.shape[2] * (1 - self.compression_ratio))
                if inv_freq is not None:
                    return native.scores_compress_rerotate(scores, keys, values, n_kept, inv_freq)[:2]
                return native.scores_compress(scores, keys, values, n_kept)[:2]
            return native.scores_compress_chunked(scores, keys, values, self.compression_ratio, self.chunk_length,
                                                  inv_freq)[:2]
        k_out, v_out, _, _ = native.finch_compress(keys, values, q, self.window_size, self.compression_ratio,
                                                   self.chunk_length, self.normalize_scores, inv_freq)
        return k_out, v_out

    def embed_token_forward_hook(self, module, input, output):
        """Forward hook of embed_tokens: finds the delimiter between the context and the question, sets window_size
        to the question's length and drops the delimiter's embedding."""
        if input[0].shape[1] > 1 and self.delimiter_token_id in input[0][0]:  # prefilling
            assert len(input[0]) == 1, "Only batch size 1 is supported."
            delim_tokens = input[0][0] == self.delimiter_token_id
            assert delim_tokens.sum() == 1, "Only one delimiter token should be present."
            context_length = int(torch.nonzero(delim_tokens)[0].item())
            self.window_size = len(input[0][0]) - 1 - context_length
            assert self.window_size > 0, "No window detected (window size must be > 0)."
            output = output[:, ~delim_tokens]
        return output

    def update_model_and_tokenizer(self, model, tokenizer, delimiter_token: str = "<|finch_sep|>"):
        """Adds the delimiter token to the tokenizer (if new) and resizes the model's embeddings. Call before the press."""
        self.delimiter_token = delimiter_token
        if delimiter_token not in tokenizer.get_vocab():
            tokenizer.add_special_tokens({"additional_special_tokens": [delimiter_token]})
        self.delimiter_token_id = tokenizer.convert_tokens_to_ids(delimiter_token)
        model.resize_token_embeddings(len(tokenizer))
        return tokenizer

    @contextmanager
    def __call__(self, model):
        if self.delimiter_token_id is None:
            raise ValueError("No delimiter token ID provided. Use the update_model_and_tokenizer method before calling "
                             "the press.")
        with super().__call__(model):
            hook = model.model.embed_tokens.register_forward_hook(self.embed_token_forward_hook)
            try:
                yield
            finally:
                hook.remove()
