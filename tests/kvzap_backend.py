"""Float64 definitions of KVzapPress's score and DMSPress's eviction (include/kvpress_b200.h, kvp_kvzap_score and
kvp_threshold_evict), and the documented bound of the kernels' score against the first."""
import math

import torch


def gelu64(t: torch.Tensor) -> torch.Tensor:
    return 0.5 * t * (1.0 + torch.erf(t / math.sqrt(2.0)))


def kvzap64(x: torch.Tensor, w1, b1, w2=None, b2=None):
    """(scores [B, Hkv, S] float64, bound E [B, Hkv, S]) of x [B, S, hidden] and the layer's weights (w2 None: the
    linear model w1 = W, b1 = b)."""
    x, w1, b1 = x.double(), w1.double(), b1.double()
    hidden = x.shape[-1]
    a = x @ w1.t() + b1                                      # [B, S, hd] (linear: [B, S, Hkv])
    A = x.abs() @ w1.abs().t() + b1.abs()
    if w2 is None:
        return a.transpose(1, 2), ((hidden + 2) * 2.0 ** -22 * A).transpose(1, 2)
    w2, b2 = w2.double(), b2.double()
    hd = w1.shape[0]
    e = (hidden + 2) * 2.0 ** -22 * A
    E_c = 1.2 * e + 2.0 ** -20 * (a.abs() + e)
    h = gelu64(a)
    s = h @ w2.t() + b2
    E = E_c @ w2.abs().t() + (hd + 260) * 2.0 ** -23 * (b2.abs() + (h.abs() + E_c) @ w2.abs().t())
    return s.transpose(1, 2), E.transpose(1, 2)


def _next16(r: torch.Tensor, up: bool) -> torch.Tensor:
    """The 16-bit neighbour of r (finite, a 16-bit dtype) towards +inf (up) or -inf, from its bit pattern."""
    bits = r.view(torch.int16).to(torch.int32) & 0xFFFF
    mag = bits & 0x7FFF
    away = (bits >= 0x8000) != up                            # the step grows the magnitude
    sign = torch.where(mag == 0, torch.full_like(bits, 0 if up else 0x8000), bits & 0x8000)
    mag = torch.where(mag == 0, torch.ones_like(mag), torch.where(away, mag + 1, mag - 1))
    return (sign | mag).to(torch.int16).view(r.dtype)


def _round_dir(v: torch.Tensor, dtype, up: bool) -> torch.Tensor:
    """v (float64) rounded to dtype towards +inf (up) or -inf, as float64."""
    r = v.to(dtype)
    fix = (r.double() < v) if up else (r.double() > v)
    return torch.where(fix, _next16(r, up).double(), r.double())


def within_bound(score: torch.Tensor, s64: torch.Tensor, E: torch.Tensor) -> torch.Tensor:
    """score (16-bit) lies in [RD(s64 - E), RU(s64 + E)]."""
    lo = _round_dir(s64 - E, score.dtype, up=False)
    hi = _round_dir(s64 + E, score.dtype, up=True)
    v = score.double()
    return (v >= lo) & (v <= hi)


def threshold_evict64(scores: torch.Tensor, n_evict: int, threshold: float, shift: int):
    """torch.where(scores[..., :n_evict] < threshold) with the last index shifted: DMSPress's eviction."""
    b, h, s = torch.where(scores[..., :n_evict] < threshold)
    return [b, h, s + shift]


def kvzap_score(hidden_states, keys, values, weights):
    """Stand-in for native.kvzap_score: the float64 definition rounded once to the cache dtype."""
    return kvzap64(hidden_states, *weights)[0].to(keys.dtype)


def kvzap_compress(hidden_states, keys, values, weights, n_kept, return_indices=False, return_scores=False):
    from tests import cpu_backend

    scores = kvzap_score(hidden_states, keys, values, weights)
    return cpu_backend.select_gather(scores, keys, values, n_kept, return_indices, return_scores)


def threshold_evict(scores, n_evict, threshold, shift):
    """Stand-in for native.threshold_evict."""
    return threshold_evict64(scores, n_evict, threshold, shift)


def install(monkeypatch):
    from kvpress_b200 import native

    for name in ("kvzap_score", "kvzap_compress", "threshold_evict"):
        monkeypatch.setattr(native, name, globals()[name])


def fp32_scores(x: torch.Tensor, w1, b1, w2=None, b2=None):
    """The surrogate evaluated in fp32 (no TF32) on x's device: (scores [B, Hkv, S] fp32, not rounded; the magnitude
    |bias| + sum of |products| of the last layer's sum, the scale of its fp32 rounding errors)."""
    saved = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        h = x.float() @ w1.float().t() + b1.float()
        mag = x.float().abs() @ w1.float().abs().t() + b1.float().abs()
        if w2 is not None:
            h = torch.nn.functional.gelu(h)
            mag = h.abs() @ w2.float().abs().t() + b2.float().abs()
            h = h @ w2.float().t() + b2.float()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = saved
    return h.transpose(1, 2), mag.transpose(1, 2)


def ulps_apart(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """How many representable 16-bit values lie between a and b (same dtype, finite): distance on the ordered grid."""
    def ordered(t):
        bits = t.view(torch.int16).to(torch.int32) & 0xFFFF
        return torch.where(bits >= 0x8000, 0x8000 - bits, bits)
    return (ordered(a) - ordered(b)).abs()
