"""A float64 stand-in for native.think_prune: the definition of include/kvpress_b200.h (kvp_think_prune) evaluated in
float64 with the fp32 rounding of the score, the library's tie rule (the lower channel is kept) and NaN rule (NaN ranks
above every number, NaNs by channel). Pure torch on any device: the host tests put it in place of the kernel, the GPU
tests compare the kernel with it."""
import torch

from kvpress_b200 import native


def scores64(keys: torch.Tensor, q_window: torch.Tensor) -> torch.Tensor:
    """qn(c) kn(c) in float64, [B, Hkv, D]: qn the mean over the G query heads of kv head j (jG ... jG+G-1) and the w
    window rows of q^2, kn the mean over the S positions of K^2."""
    B, H, S, D = keys.shape
    G = q_window.shape[1] // H
    qn = q_window.double().square().mean(dim=2).view(B, H, G, D).mean(dim=2)
    kn = keys.double().square().mean(dim=2)
    return qn * kn


def pruned_mask(scores: torch.Tensor, n_pruned: int) -> torch.Tensor:
    """True on the channels outside the D - n_pruned largest scores of each row (ties: the lower channel is kept; NaN
    above every number, NaNs by channel)."""
    D = scores.shape[-1]
    a, b = scores.unsqueeze(-1), scores.unsqueeze(-2)  # a: the other channel c', b: channel c
    lower = torch.ones(D, D, dtype=torch.bool, device=scores.device).triu(1)  # [c', c]: c' < c
    an, bn = a.isnan(), b.isnan()
    beats = (a > b) | ((a == b) & lower) | (an & ~bn) | (an & bn & lower)
    return beats.sum(dim=-2) >= D - n_pruned


def think_prune64(keys: torch.Tensor, q_window: torch.Tensor, n_pruned: int, return_pruned: bool = False,
                  return_scores: bool = False):
    """native.think_prune's contract: keys zeroed in place on the pruned channels; (keys, pruned, scores)."""
    if n_pruned == 0:
        return keys, None, None
    scores = scores64(keys, q_window).float()
    mask = pruned_mask(scores, n_pruned)
    keys.masked_fill_(mask.unsqueeze(2), 0.0)
    B, H, D = scores.shape
    pruned = mask.nonzero()[:, 2].view(B, H, n_pruned).to(torch.int32) if return_pruned else None
    return keys, pruned, scores if return_scores else None


def install(monkeypatch):
    monkeypatch.setattr(native, "think_prune", think_prune64)
