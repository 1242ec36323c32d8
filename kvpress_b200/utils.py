"""Model introspection helpers used by the presses (host side, torch plumbing).

Mirrors the two helpers of the reference that sit on the hot path
(`kvpress/utils.py:12-53` get_prerope_query_states, `:104-114`
extract_keys_and_values). Llama-like (`q_proj`) and Qwen3/Gemma3 (`q_proj` + `q_norm`) attention
modules are supported; Phi3's fused `qkv_proj` is sliced. Quantized caches are out of scope.
"""
from __future__ import annotations

import torch
from torch import nn


def get_prerope_query_states(module: nn.Module, hidden_states: torch.Tensor) -> torch.Tensor:
    """Project `hidden_states` [B, L, hidden] to pre-RoPE queries [B, Hq, L, D] with the layer's own weights."""
    batch, length, _ = hidden_states.shape
    n_heads = module.config.num_attention_heads
    head_dim = module.head_dim
    if hasattr(module, "qkv_proj"):  # Phi3-style fused projection: queries come first
        q = module.qkv_proj(hidden_states)[..., : n_heads * head_dim]
    elif hasattr(module, "q_proj"):
        q = module.q_proj(hidden_states)
    else:
        raise NotImplementedError(f"no query projection found on {module.__class__.__name__}")
    q = q.view(batch, length, n_heads, head_dim).transpose(1, 2)
    q_norm = getattr(module, "q_norm", None)
    if q_norm is not None:  # Qwen3 / Gemma3 normalise per head before RoPE
        q = q_norm(q)
    return q


def extract_keys_and_values(cache, layer_idx: int) -> tuple[torch.Tensor, torch.Tensor]:
    """Return the (keys, values) tensors [B, Hkv, S, D] a DynamicCache holds for one layer."""
    layer = cache.layers[layer_idx]
    if hasattr(layer, "_quantized_keys"):
        raise NotImplementedError("kvpress_b200 does not handle QuantizedCache layers (out of scope)")
    return layer.keys, layer.values


def rotate_half(x: torch.Tensor) -> torch.Tensor:
    half = x.shape[-1] // 2
    return torch.cat((-x[..., half:], x[..., :half]), dim=-1)


def apply_rope(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    """x: [B, H, L, D]; cos/sin: [B or 1, L, D] (the `position_embeddings` HF passes to attention)."""
    return x * cos.unsqueeze(1) + rotate_half(x) * sin.unsqueeze(1)


def last_query(module: nn.Module, hidden_states: torch.Tensor, kwargs: dict) -> torch.Tensor:
    """RoPE'd query of the last position of `hidden_states`, [B, Hq, D] (TOVAPress's score, CAMPress's decode step)."""
    q = get_prerope_query_states(module, hidden_states[:, -1:])
    cos, sin = kwargs["position_embeddings"]
    return apply_rope(q, cos[:, -1:], sin[:, -1:])[:, :, 0].contiguous()
