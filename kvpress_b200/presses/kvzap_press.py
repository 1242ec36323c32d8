"""KVzapPress: scores from a small per-layer surrogate model of the hidden states (https://arxiv.org/abs/2601.07891).

API mirror of `kvpress/presses/kvzap_press.py`. Each layer's score is a linear map or a two-layer GELU MLP of the
attention module's input hidden states, one output per kv head; it reads no queries, attention weights or K / V, so it
runs under every attention implementation and inside every wrapper press. `KVzapConfig` / `KVzapModel` load the
published `nvidia/KVzap-*` checkpoints (config fields `input_dim, output_dim, hidden_dim, n_modules`; state-dict keys
`layers.{i}.weight|bias` for the linear model, `layers.{i}.0.*` and `layers.{i}.2.*` for the MLP).

Differences from the reference: the weights are cast to the cache dtype once per (layer, device, dtype), not on every
call; the model is evaluated by the sm_90a kernels of csrc/kvzap.cu with fp32 sums and one rounding of the score,
instead of Linear -> GELU -> Linear in the cache dtype. Shapes outside those kernels score with cuBLAS in fp32
(logged once); selection stays on the sm_90a kernels. The hidden states must cover the positions being scored:
under DecodingPress, whose buffer holds fewer hidden states than the cache has positions, score() raises (the
reference's topk over the shorter score row fails there too).
"""
from __future__ import annotations

import logging
from dataclasses import dataclass, field
from typing import Literal, Optional

import torch
import torch.nn as nn
from transformers import PretrainedConfig, PreTrainedModel

from kvpress_b200 import native
from kvpress_b200.presses.scorer_press import ScorerPress

logger = logging.getLogger(__name__)
_warned: set = set()


class KVzapConfig(PretrainedConfig):
    """One surrogate per layer (n_modules) from input_dim hidden features to output_dim kv heads; hidden_dim None is
    the linear model, an int the width of the MLP."""

    model_type = "kvzap"

    def __init__(self, input_dim: int = 0, output_dim: int = 0, n_modules: int = 0, hidden_dim: Optional[int] = None,
                 **kwargs):
        super().__init__(**kwargs)
        self.input_dim = input_dim
        self.output_dim = output_dim
        self.hidden_dim = hidden_dim
        self.n_modules = n_modules


def _surrogate(config: KVzapConfig) -> nn.Module:
    if config.hidden_dim is None:
        return nn.Linear(config.input_dim, config.output_dim)
    return nn.Sequential(nn.Linear(config.input_dim, config.hidden_dim), nn.GELU(),
                         nn.Linear(config.hidden_dim, config.output_dim))


class KVzapModel(PreTrainedModel):
    """`layers[i]` maps layer i's hidden states [..., input_dim] to its kv-head scores [..., output_dim]."""

    config_class = KVzapConfig

    def __init__(self, config: KVzapConfig):
        super().__init__(config)
        self.all_tied_weights_keys = {}
        self.layers = nn.ModuleList(_surrogate(config) for _ in range(config.n_modules))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x [N, n_modules, input_dim] -> [N, n_modules, output_dim]."""
        return torch.stack([layer(x[:, i]) for i, layer in enumerate(self.layers)], dim=1)


def layer_weights(layer: nn.Module) -> tuple:
    """(w1, b1, w2, b2) of an MLP surrogate, (W, b, None, None) of a linear one, as stored."""
    if isinstance(layer, nn.Linear):
        return layer.weight, layer.bias, None, None
    return layer[0].weight, layer[0].bias, layer[2].weight, layer[2].bias


class _fp32_matmul:
    """Keeps the fallback's GEMMs in full fp32 even where TF32 is enabled."""

    def __enter__(self):
        self.saved = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = False

    def __exit__(self, *exc):
        torch.backends.cuda.matmul.allow_tf32 = self.saved


def torch_scores(hidden_states: torch.Tensor, weights: tuple) -> torch.Tensor:
    """The surrogate with cuBLAS in fp32 (shapes outside the kernels): [B, Hkv, S] in the hidden states' dtype."""
    w1, b1, w2, b2 = (None if w is None else w.float() for w in weights)
    x = hidden_states.float()
    with _fp32_matmul():
        out = torch.addmm(b1, x.reshape(-1, x.shape[-1]), w1.t())
        if w2 is not None:
            out = torch.addmm(b2, torch.nn.functional.gelu(out), w2.t())
    return out.view(x.shape[0], x.shape[1], -1).transpose(1, 2).to(hidden_states.dtype)


@dataclass
class KVzapPress(ScorerPress):
    """Prunes the positions the layer's surrogate model scores lowest. model_type "linear" or "mlp"; meant to be used
    inside DMSPress (threshold eviction), and usable wherever a ScorerPress is."""

    model_type: Literal["linear", "mlp"] = "mlp"
    kvzap_model_name: Optional[str] = field(default=None, init=False)
    kvzap_model: Optional[KVzapModel] = field(default=None, repr=False)
    _cast: dict = field(default_factory=dict, init=False, repr=False)

    def post_init_from_model(self, model):
        """Loads nvidia/KVzap-{model_type}-{model name} from the Hub, as the reference does, whenever that name differs
        from the one loaded last. A kvzap_model set by the user (kvzap_model_name None) is kept."""
        if self.kvzap_model is not None and self.kvzap_model_name is None:
            return
        name = f"nvidia/KVzap-{self.model_type}-{model.config.name_or_path.split('/')[-1]}"
        if name != self.kvzap_model_name:
            self.kvzap_model = KVzapModel.from_pretrained(name)
            self.kvzap_model_name = name

    def weights(self, layer_idx: int, like: torch.Tensor) -> tuple:
        """Layer layer_idx's weights in like's dtype on like's device, cast once per surrogate model."""
        if self.kvzap_model is None:
            raise RuntimeError("KVzapPress has no surrogate model: set kvzap_model or call post_init_from_model")
        if self._cast.get("model") is not self.kvzap_model:  # a replaced model drops every cast of the old one
            self._cast = {"model": self.kvzap_model}
        key = (layer_idx, like.device, like.dtype)
        hit = self._cast.get(key)
        if hit is None:
            hit = self._cast[key] = tuple(
                None if w is None else w.detach().to(like.device, like.dtype).contiguous()
                for w in layer_weights(self.kvzap_model.layers[layer_idx]))
        return hit

    def _scored_rows(self, hidden_states: torch.Tensor, keys: torch.Tensor) -> torch.Tensor:
        if hidden_states.shape[1] != keys.shape[2]:
            raise ValueError(f"KVzapPress scores the positions of its hidden states: got {hidden_states.shape[1]} "
                             f"hidden states for {keys.shape[2]} cached positions")
        return hidden_states.to(keys.dtype)

    def _on_kernels(self, weights: tuple, keys: torch.Tensor) -> bool:
        hd = 0 if weights[2] is None else weights[0].shape[0]
        if native.kvzap_supported(weights[0].shape[1], hd, keys.shape[1]):
            return True
        key = (weights[0].shape[1], hd, keys.shape[1])
        if key not in _warned:
            _warned.add(key)
            logger.warning(f"KVzapPress: hidden {key[0]} / width {hd} / {key[2]} kv heads is outside the sm_90a "
                           "kernels; scoring with cuBLAS in fp32")
        return False

    def score(self, module: nn.Module, hidden_states, keys: torch.Tensor, values: torch.Tensor, attentions,
              kwargs) -> torch.Tensor:
        x = self._scored_rows(hidden_states, keys)
        w = self.weights(module.layer_idx, keys)
        if not self._on_kernels(w, keys):
            return torch_scores(x, w)
        return native.kvzap_score(x, keys, values, w)

    def _fused_compress(self, module, hidden_states, keys, values, attentions, kwargs, n_kept):
        if self._score_is_overridden(KVzapPress):
            return None
        x = self._scored_rows(hidden_states, keys)
        w = self.weights(module.layer_idx, keys)
        if not self._on_kernels(w, keys):
            return None  # score() runs the cuBLAS fallback; the generic selection follows
        k_out, v_out, _, _ = native.kvzap_compress(x, keys, values, w, n_kept)
        return k_out, v_out
