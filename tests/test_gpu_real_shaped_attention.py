"""The softmax scorers (SnapKV, ExpectedAttention with and without covariance, ObservedAttention, NonCausalAttention,
Finch) on caches shaped like a trained model's, against float64.

The other scorer tests draw K and q from N(0, 1), so raw logits are O(1) and the fp32 error of a logit, which grows with
sum_i |q_i k_i|, stays far below half an ulp of the cache dtype. A trained model's cache has attention sinks (keys 0-3
taking most of every query's mass), massive-activation channels (a few low-frequency RoPE channels 10-50x the others in
q and k, a large sum_i |q_i k_i| for a small net logit) and peaked rows (most probabilities tiny, many fp16 scores +0).
`real_shaped` builds such caches from a seed; the cases below run every scorer on them.

The bar. A position passes if either
  1. its score is within 1 ulp of the float64 score rounded once (with the ftz rule of the scorer), or
  2. it lies in [RD(ref - E_s |ref|), RU(ref + E_s |ref|)] in the cache dtype,
where E_s is an a-priori bound on the kernel's fp32 error relative to the score, computed in float64 from the inputs
(NonCausalAttention: the absolute bound of tests/test_gpu_non_causal_attention.py). The row-bias bar of the other sweeps
applies to the rows whose largest E_s is below a quarter of it; forced positions hold round(max + 1) bitwise. That
gate is strict: the bias bound of a row of n positions is 8 u16 / sqrt(12 n), and on these caches E_s (of order 1e-5 to
1e-4 at a few thousand positions) stays above a quarter of it, so few or no rows of this file are held to the bias bar
(the [measured] lines count them). The bias of Gaussian rows is held by the other sweeps.

E_s, derived from the kernels' operations. u = 2^-24 (fp32). Products of two 16-bit values are exact in fp32, and a
wgmma sums D of them in fp32, so a raw logit y = q.k carries |dy| <= gamma_D A, A = sum_i |q_i k_i|,
gamma_D = (D + 1) u.

SnapKV, ObservedAttention, Finch (qk_tiles.cuh). c = RN(scaling log2 e); pass 1 keeps the row's (m, Z) online, pass 2
recomputes the product (another MMA shape: its own rounding, within the same gamma_D A of y) and adds
P = ex2(fma(y, c, cb)), cb = -(m c) - log2f(Z) [+ log2f(c_i), Finch's normalisation]. The row max cancels between Z and
the exponent up to its roundings. In log2 units, with M the row's largest logit and x = log2 P [+ log2 c_i]:
  - the exponent: c gamma_D A_s (pass 2) + u (|c y_s| + 3 |c M| + 5 log2 Z + 3 log2 c_i + |x_s|);
  - ex2.approx: 2^-22 relative;
  - Z: the P-weighted mean of its terms' exponent errors, c gamma_D A_j + u (|c y_j| + |c (y_j - M)|),
    + u |c M| + 2^-22,
    and its chain: per tile four chains of 8 terms and one rescale by ex2((m - m') c), the quad and part merges, at most
    2 n_t + 2 rescales and 2 n_t + 12 additions (n_t tiles in the row's causal span), (12 n_t + 22) u, plus the
    rescale arguments, which telescope to 4 u c (max |y|).
The relative error of P is ln 2 times the exponent's plus the two 2^-22 and Z's. The column sum of P w_i over G n_q rows
adds (20 + G ceil(n_q / 128)) u (per 128-row chunk 16 + 1 terms, the chunks, the quad sum), flushed terms below 2^-126
at most G n_q 2^-126 w_max, and the finalisation (SnapKV: the box filter and 1/(G w), (k + 4) u; ObservedAttention and
Finch: one division and one product, 4 u).

ExpectedAttention (expected_attention.cu). t = sum_n k_n (Y_n + RN(2 sqrt(D)) mu_n), Y = K Sigma^T on wgmma; the
logit is t / (2D). Y carries gamma_D |Sigma| |k|; the add, the bias product and the fma chain of D / 4 + 2 terms add
(D / 4 + 6) u of sum_n |k_n| (|Y_n| + |b_n|). So
dl <= gamma_E (|k|^T |Sigma| |k| / (2D) + |mu|.|k| / sqrt(D)) + 3 u |l|,
gamma_E = (5 D / 4 + 6) u; the covariance-free GEMV (8-term fma chains, log2(LPR) shuffles, one product with 1/sqrt(D))
is within the same. __expf(x) is accurate to (2 + 1.173 |x|) ulp; every running (m, z) update costs two roundings and a
rescale, at most 2 ceil(S / 128) + 64 of them on any chain (tiles or lanes, warp, CTA, parts), the rescale arguments
telescoping to 4 (max l - min l) over the four merge levels. p = mean_g __expf(l - m) / Z adds (G + 4) u,
(p + eps) ||v|| adds u and (D + 4) u for the fp32 norm, and each flushed __expf at most 2^-126. E_s is that sum, times
1.01 for the second-order terms.

Each part is an upper bound of the operation as the kernel orders it; none is fitted to a measurement.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import press_oracle as O
from tests import gpu_support as GS
from tests import non_causal_attention_backend as NB
from tests.gpu_support import (assert_compress, ea_ref64, ea_schedule, nca_ref, oa_ref64, scores64, snap_parts,
                               snap_ref64, ulp16_diff, UNIT_ROUNDOFF, U32, BIAS_MIN_N, _forced_head, _forced_tail,
                               _name, _native)

gpu = pytest.mark.gpu
DEV = "cuda:0"
BF16, FP16 = torch.bfloat16, torch.float16
LOG2E = 1.0 / math.log(2.0)
LN2 = math.log(2.0)
TINY32 = 2.0 ** -126


# ---------------------------------------------------------------------------------------------------
# 1. real-shaped caches
# ---------------------------------------------------------------------------------------------------
def _rope(x, pos, inv_freq):
    ang = pos.double()[:, None] * inv_freq.double()[None, :]
    cos, sin = torch.cat((ang.cos(), ang.cos()), -1), torch.cat((ang.sin(), ang.sin()), -1)
    return x * cos.to(x) + O.rotate_half(x) * sin.to(x)


def massive_channels(D: int):
    """the first channel of the two lowest-frequency RoPE pairs"""
    return [D // 2 - 1, D // 2 - 3]


class RealShaped:
    """K, V [B, Hkv, S, D] and the queries at every position q [B, Hkv G, S, D], 16-bit; the scorers' query operands."""

    def __init__(self, k, v, q):
        self.k, self.v, self.q = k, v, q

    def window(self, w: int):
        """SnapKV and Finch: the queries at positions S - w .. S - 1"""
        return self.q[:, :, -w:].contiguous()

    def last(self):
        """TOVAPress: the last query, as ExpectedAttention's mu (covariance-free, n_sink 0, no value norms)"""
        return self.q[:, :, -1].contiguous()

    def ea_stats(self, regime: str):
        """(mu, Sigma) in the cache dtype: the float64 mean and covariance of the queries, rounded once. "mean": as
        they are (the massive channels sit in mu); "variance": mu shrunk to a quarter and Sigma given a large eigenvalue
        along the first massive channel at the last position."""
        q = self.q.double()
        mu = q.mean(2)
        d = q - mu[:, :, None]
        cov = d.transpose(-1, -2) @ d / q.shape[2]
        if regime == "variance":
            D = q.shape[-1]
            e = torch.zeros(D, dtype=torch.float64, device=q.device)
            e[massive_channels(D)[0]] = 1.0
            amp = float(q[..., massive_channels(D)[0]].abs().mean())
            cov = cov + (8.0 * D / max(1.0, amp) ** 2) * torch.outer(e, e)
            mu = 0.25 * mu
        return mu.to(self.k.dtype), cov.to(self.k.dtype)


def real_shaped(B, Hkv, G, S, D, dtype, seed, *, sink=0.0, massive=0.0, peak=1.5, theta=500000.0, device=DEV):
    """A seeded cache with a trained model's shape. Pre-RoPE q and k get RoPE (Llama-3 theta) at their positions.
    - peak: the std of the bulk's scaled logits q.k / sqrt(D) (queries of std `peak` per channel, 64 % of their variance
      along one direction per kv head, shared by its G heads and every position);
    - massive: the amplitude of the two lowest-frequency channel pairs in q and k (2 % jitter), a large sum |q_i k_i|
      whose net logit is nearly the same for every key;
    - sink: the scaled-logit margin of keys 0..3 over the bulk along the mean query direction of each kv head;
    - values: row norms log-normal (sigma 0.7), the sink rows 20x smaller."""
    g = torch.Generator(device=device).manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device=device, dtype=torch.float64)  # noqa: E731
    Hq = Hkv * G
    pos = torch.arange(S, device=device)
    inv = 1.0 / (theta ** (torch.arange(0, D, 2, dtype=torch.float64, device=device) / D))
    k0 = rn(B, Hkv, S, D)
    direction = rn(B, Hkv, 1, 1, D)
    q0 = peak * (0.6 * rn(B, Hkv, G, S, D) + 0.8 * direction) / math.sqrt(0.36 + 0.64)
    q0 = q0.reshape(B, Hq, S, D)
    if massive:
        for ch in massive_channels(D):
            k0[..., ch] = massive * (1 + 0.02 * rn(B, Hkv, S))
            q0[..., ch] = massive * (1 + 0.02 * rn(B, Hq, S))
    k, q = _rope(k0, pos, inv), _rope(q0, pos, inv)
    if sink and S > 4:
        qg = q.reshape(B, Hkv, G * S, D)
        qbar = qg.mean(2)                                                              # [B, Hkv, D]
        qn = qbar.norm(dim=-1)[..., None, None]
        qhat = qbar[:, :, None] / qn
        # mean raw logit of the bulk; the sink keys lose their component along qhat and get one whose mean logit is
        # that plus sink sqrt(D)
        bulk = (qbar[:, :, None] * k[:, :, 4:]).sum(-1).mean(-1)[..., None, None]
        ks = k[:, :, :4] - (k[:, :, :4] * qhat).sum(-1, keepdim=True) * qhat
        k[:, :, :4] = ks + (bulk + sink * math.sqrt(D)) / qn * qhat
    v = torch.exp(0.7 * rn(B, Hkv, S, 1)) * rn(B, Hkv, S, D)
    v[:, :, :4] *= 0.05
    return RealShaped(k.to(dtype), v.to(dtype), q.to(dtype))


# ---------------------------------------------------------------------------------------------------
# 2. the bounds E_s (module docstring), float64 on the inputs' device
# ---------------------------------------------------------------------------------------------------
def colsum_bound64(k, q, scaling, row_w, normalize_log2=None, rows=None):
    """(col, err), float64 [B, H, S]: col_s = sum_{g, i} row_w[i] P_{g i}(s) of the causal softmax of query row i
    (position S - n_q + i), err_s the bound on its fp32 evaluation's absolute error, before the finalisation.
    normalize_log2: [n_q] log2 c_i that Finch folds into the exponent (0 elsewhere)."""
    B, H, S, D = k.shape
    Hq, n_q = q.shape[1], q.shape[2]
    G, off = Hq // H, S - n_q
    c = scaling * LOG2E
    lam = c * (D + 1) * U32
    u = U32
    w = row_w.double().to(k.device)
    lc = torch.zeros(n_q, dtype=torch.float64, device=k.device) if normalize_log2 is None else normalize_log2
    rows = rows or max(1, (1 << 24) // S)
    col = torch.zeros(B, H, S, dtype=torch.float64, device=k.device)
    err = torch.zeros_like(col)
    spos = torch.arange(S, device=k.device)
    for b in range(B):
        for h in range(H):
            kk = k[b, h].double()
            ka = kk.abs()
            for gq in range(G):
                qh = q[b, h * G + gq].double()
                for i0 in range(0, n_q, rows):
                    i1 = min(n_q, i0 + rows)
                    qq = qh[i0:i1]
                    rpos = torch.arange(off + i0, off + i1, device=k.device)
                    masked = spos[None, :] > rpos[:, None]
                    y = (qq @ kk.T).masked_fill(masked, -math.inf)
                    A = (qq.abs() @ ka.T).masked_fill(masked, 0.0)
                    M = y.amax(-1, keepdim=True)
                    t = c * (y - M)                                                    # log2, <= 0
                    e = torch.exp2(t)
                    Z = e.sum(-1, keepdim=True)
                    P = e / Z
                    L = torch.log2(Z)
                    yf = torch.where(masked, 0.0, y)
                    tf = torch.where(masked, 0.0, t)
                    cy, cM = (c * yf).abs(), (c * M).abs()
                    li = lc[i0:i1, None]
                    x = (tf - L + li).abs()
                    n_t = torch.div(rpos + 1 + 127, 128, rounding_mode="floor").double()[:, None]
                    ymax = yf.abs().amax(-1, keepdim=True)
                    chain = (12 * n_t + 22) * u + 4 * u * c * ymax
                    eZ = LN2 * ((P * (lam * A + u * (cy - tf))).sum(-1, keepdim=True) + u * cM) + 2.0 ** -22 + chain
                    eP = LN2 * (lam * A + u * (cy + 3 * cM + 5 * L + 3 * li + x)) + 2.0 ** -22 + 2.0 ** -22 + eZ
                    wi = w[i0:i1, None]
                    col[b, h] += (wi * P).sum(0)
                    err[b, h] += (wi * P * eP).sum(0)
    depth = 20 + G * -(-n_q // 128)
    err += depth * u * col + G * n_q * float(w.max()) * TINY32
    return col, err


def snap_bound64(k, q, window, kernel_size):
    """E_s of SnapKV (relative), [B, H, S]; 0 on the window"""
    B, H, S, D = k.shape
    G = q.shape[1] // H
    col, err = colsum_bound64(k, q, D ** -0.5, torch.full((window,), 1.0 / (G * window)))
    n = S - window
    score, abs_err = (F.avg_pool1d(x[..., :n].reshape(B * H, 1, n), kernel_size, 1, kernel_size // 2).reshape(B, H, n)
                      for x in (col, err))
    E = torch.zeros(B, H, S, dtype=torch.float64, device=k.device)
    E[..., :n] = 1.01 * (abs_err / score.clamp_min(1e-300) + (kernel_size + 4) * U32)
    return E


def finch_bound64(k, q, window, normalize):
    B, H, S, D = k.shape
    G = q.shape[1] // H
    rpos = torch.arange(S - window, S, device=k.device, dtype=torch.float64)
    wts = (rpos if normalize else torch.ones_like(rpos)) / (G * window)
    col, err = colsum_bound64(k, q, D ** -0.5, wts, torch.log2(rpos) if normalize else None)
    E = torch.zeros(B, H, S, dtype=torch.float64, device=k.device)
    E[..., :S - window] = 1.01 * (err / col.clamp_min(1e-300) + 4 * U32)[..., :S - window]
    return E


def oa_bound64(k, q, scaling):
    n_q = q.shape[2]
    col, err = colsum_bound64(k, q, scaling, torch.ones(n_q))
    return 1.01 * (err / col.clamp_min(1e-300) + 4 * U32)


def ea_bound64(k, v, mu, cov, eps, n_sink, use_vnorm):
    """E_s of ExpectedAttention (relative), [B, H, S]; 0 on the sinks"""
    B, H, S, D = k.shape
    G = mu.shape[1] // H
    u = U32
    gam = (5 * D / 4 + 6) * u
    eps = float(torch.tensor(eps, dtype=torch.float32))
    n_upd = 2 * -(-S // 128) + 64
    E = torch.zeros(B, H, S, dtype=torch.float64, device=k.device)
    if S <= n_sink:
        return E
    for b in range(B):
        for h in range(H):
            kk = k[b, h, n_sink:].double()
            ka = kk.abs()
            p = torch.zeros(S - n_sink, dtype=torch.float64, device=k.device)
            pe = torch.zeros_like(p)
            for gq in range(G):
                m = mu[b, h * G + gq].double()
                lg = kk @ m / math.sqrt(D)
                T = ka @ m.abs() / math.sqrt(D)
                if cov is not None:
                    C = cov[b, h * G + gq].double()
                    lg = lg + ((kk @ C) * kk).sum(-1) / (2 * D)
                    T = T + ((ka @ C.abs()) * ka).sum(-1) / (2 * D)
                dl = gam * T + 3 * u * lg.abs()
                x = lg - lg.max()
                P = torch.softmax(lg, -1)
                ex = u * x.abs() + (4 + 2.346 * x.abs()) * u
                chain = n_upd * 6 * u + 2.346 * u * 4 * float(lg.max() - lg.min())
                eZ = (P * (dl + ex)).sum() + chain
                eP = dl + ex + 4 * u + eZ
                p += P
                pe += P * eP
            p, pe = p / G, pe / G + (G + 4) * u * p / G + TINY32  # its G terms each flushed below 2^-126
            if use_vnorm:
                E[b, h, n_sink:] = 1.01 * ((pe + u * (p + eps)) / (p + eps) + (D + 5) * u)
            else:
                E[b, h, n_sink:] = 1.01 * (pe / p.clamp_min(1e-300))
    return E


# ---------------------------------------------------------------------------------------------------
# the bar
# ---------------------------------------------------------------------------------------------------
def _step16(x: torch.Tensor, up: bool) -> torch.Tensor:
    """the next 16-bit value above (below) x, as float64 (from +-0 the smallest subnormal of that side)"""
    b = x.contiguous().view(torch.int16).to(torch.int32) & 0xFFFF
    neg = b >= 0x8000
    mag = b & 0x7FFF
    grow = neg != up                                   # moving away from zero
    new_mag = torch.where(grow, mag + 1, mag - 1)
    new_b = torch.where(mag == 0, torch.where(torch.tensor(up, device=x.device), 0x0001, 0x8001),
                        torch.where(new_mag < 0, 0, (b & 0x8000) | new_mag))
    return new_b.to(torch.int16).view(x.dtype).double()


def assert_real(got, ref, E, forced, what: str, ftz: bool = False, bias: bool = True, absolute: bool = False) -> dict:
    """Conditions 1 and 2 of the module docstring, the row-bias bar where E is small, the sentinel. E is relative to
    |ref| unless `absolute`. Returns the measured statistics."""
    dtype = got.dtype
    ref, E, forced = ref.to(got.device), E.to(got.device), forced.to(got.device)
    g, r = got[..., ~forced], ref[..., ~forced]
    e = E[..., ~forced] * (1.0 if absolute else r.abs())
    assert torch.isfinite(g).all(), f"{what}: non-finite scores"
    d = ulp16_diff(g, r.to(dtype))
    c1 = d <= 1
    if ftz:
        c1 |= (r < 2.0 ** -126) & (g == 0)
    c2 = (_step16(g, True) > r - e) & (_step16(g, False) < r + e)
    ok = c1 | c2
    if not ok.all():
        i = (~ok).nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int((~ok).sum())} positions beyond both bars, first at {i}: got "
                             f"{float(g[tuple(i)])} ref {float(r[tuple(i)])} E {float(e[tuple(i)]):.3e} "
                             f"({int(d[tuple(i)])} ulp)")
    rel_e = E[..., ~forced] if not absolute else e / r.abs().amax(-1, keepdim=True).clamp_min(1e-300)
    nrm = r.abs() >= torch.finfo(dtype).tiny  # the largest E_s among scores in the normal range of the dtype
    stats = {"max_e": float(rel_e[nrm].max()) if nrm.any() else 0.0,
             "e_only": float((~c1).float().mean()) if c1.numel() else 0.0, "bias": 0.0, "bias_rows": 0}
    if bias:
        normal = (r.abs() >= torch.finfo(dtype).tiny) & c1
        n = normal.sum(-1)
        rel = torch.where(normal, (g.double() - r) / r, torch.zeros_like(r))
        mean = rel.sum(-1) / n.clamp_min(1)
        bound = 8 * UNIT_ROUNDOFF[dtype] / torch.sqrt(12.0 * n.clamp_min(1).double())
        rows = (n >= BIAS_MIN_N) & (torch.where(normal, rel_e, 0.0).amax(-1) <= bound / 4)
        stats["bias_rows"] = int(rows.sum())
        ratio = (mean.abs() / bound)[rows]
        if ratio.numel():
            stats["bias"] = float(ratio.max())
            assert (ratio <= 1).all(), f"{what}: row bias {stats['bias']:.2f}x its bound"
    if forced.any():
        sentinel = (g.float().max() + 1).to(dtype)
        assert (got[..., forced] == sentinel).all(), f"{what}: forced positions are not round(max + 1)"
    print(f"[measured] {what}: max E {stats['max_e']:.2e}, share needing the E interval {stats['e_only']:.2e}, "
          f"max ulp {int(d.max()) if d.numel() else 0}, rows held to the bias bar {stats['bias_rows']}, "
          f"worst row bias {stats['bias']:.3f} of its bound")
    return stats


# ---------------------------------------------------------------------------------------------------
# CPU: the inputs are what they claim, and E_s is consistent with the existing bars and with an fp32 evaluation
# ---------------------------------------------------------------------------------------------------
def _window_softmax64(r: RealShaped, w: int):
    """[B, Hq, w, S] float64 causal softmax of the window rows"""
    k, q = r.k.double(), r.window(w).double()
    B, H, S, D = k.shape
    G = q.shape[1] // H
    y = (q.reshape(B, H, G * w, D) @ k.transpose(-1, -2)).reshape(B, H * G, w, S)
    rp = torch.arange(S - w, S)
    y = y.masked_fill(torch.arange(S)[None, :] > rp[:, None], -math.inf)
    return torch.softmax(y / math.sqrt(D), -1), y


@pytest.mark.parametrize("sink,massive,peak", [(0, 0, 1.5), (10, 0, 1.5), (25, 8, 1.5), (0, 30, 4), (0, 0, 12)])
def test_real_shaped_inputs_are_what_they_claim(sink, massive, peak):
    S, w, D = 2048, 64, 64
    r = real_shaped(1, 2, 2, S, D, FP16, 3, sink=sink, massive=massive, peak=peak, device="cpu")
    P, y = _window_softmax64(r, w)
    share = float(P[..., :4].sum(-1).mean())
    top1 = float(P.amax(-1).median())
    ymax = float(torch.where(torch.isinf(y), 0.0, y).abs().max())
    zeros = int((snap_ref64(r.window(w), r.k, w, 1)[..., :S - w].to(FP16) == 0).sum())
    print(f"[measured] sink {sink} massive {massive} peak {peak}: sink share {share:.3f}, median top-1 {top1:.3f}, "
          f"max |raw logit| {ymax:.0f}, fp16 +0 scores {zeros}")
    assert share >= {0: 0.0, 10: 0.8, 25: 0.99}[sink] and (sink or share < 0.02)
    if peak >= 12:
        assert top1 >= 0.8 and zeros >= 1000           # peaked rows, and a plateau of +0 scores
    if massive:
        assert ymax >= 2 * massive ** 2 * 0.9          # the massive channels' product: two pairs of massive^2
    else:
        assert ymax <= 60 * peak + (sink + 10) * math.sqrt(D)
    if peak <= 1.5 and not sink:
        assert top1 < 0.1 and zeros == 0


def _half_ulp_rel(dtype):
    return UNIT_ROUNDOFF[dtype] / 4  # half an ulp relative to the value, at the top of a binade


def test_bound_on_the_gaussian_inputs_is_below_half_an_ulp(monkeypatch):
    """On the inputs of the other sweeps (N(0, 1) keys, 1.5 N(0, 1) queries), E_s stays below half an ulp everywhere:
    there the 1-ulp bar alone was sound, as their docstrings argue."""
    monkeypatch.setattr(GS, "DEV", "cpu")
    for dt in (BF16, FP16):
        k, v, q = GS.snap_inputs(1, 2, 4, 2500, 128, 64, dt, 1)
        assert float(snap_bound64(k, q, 64, 5).max()) < _half_ulp_rel(dt)
        assert float(finch_bound64(k, q, 64, True).max()) < _half_ulp_rel(dt)  # test_gpu_finch's inputs: the same law
        k, v, mu, cov = GS.ea_inputs(1, 2, 4, 2500, 128, dt, 2)
        assert float(ea_bound64(k, v, mu, cov, 0.0, 4, True).max()) < _half_ulp_rel(dt)
        assert float(ea_bound64(k, v, mu, None, 0.0, 4, False).max()) < _half_ulp_rel(dt)
        k, v, q = GS.oa_inputs(1, 1, 2, 1000, 1000, 64, dt, 3)
        assert float(oa_bound64(k, q, 64 ** -0.5).max()) < _half_ulp_rel(dt)


FP32_CASES = [(0, 30, 4), (25, 8, 1.5), (10, 0, 12)]


@pytest.mark.parametrize("sink,massive,peak", FP32_CASES)
def test_fp32_evaluation_stays_inside_the_bound(sink, massive, peak):
    """torch's float32 evaluation of each formula (its own GEMM and summation order) is within E_s of float64: SnapKV,
    Finch with and without its position weights, ObservedAttention, ExpectedAttention in both regimes and the
    covariance-free TOVA call. (NonCausalAttention's bound is the one tests/test_gpu_non_causal_attention.py holds
    its kernel to.)"""
    S, D, w = 700, 64, 40
    r = real_shaped(1, 2, 2, S, D, BF16, 5, sink=sink, massive=massive, peak=peak, device="cpu")
    k, q = r.k, r.window(w)

    def inside(f32, ref, E, what):
        fin = torch.isfinite(ref) & (E > 0)
        bad = (f32.double() - ref).abs()[fin] > (E * ref.abs())[fin]
        assert not bad.any(), f"{what}: {int(bad.sum())} fp32 values outside E_s"

    inside(O.snapkv_scores_fp32(q, k, w, 5), snap_ref64(q, k, w, 5), snap_bound64(k, q, w, 5), "snapkv")
    qa = r.q
    y = (qa.float().reshape(1, 2, 2 * S, D) @ k.float().transpose(-1, -2)).reshape(1, 4, S, S) * D ** -0.5
    y = y.masked_fill(torch.arange(S)[None, :] > torch.arange(S)[:, None], -math.inf)
    col = torch.softmax(y, -1).sum(2).reshape(1, 2, 2, S).sum(2)
    oa32 = col / (2 * torch.arange(S, 0, -1).to(BF16).float())
    inside(oa32, oa_ref64(k, qa, D ** -0.5), oa_bound64(k, qa, D ** -0.5), "observed attention")
    for normalize in (False, True):
        yw = (q.float().reshape(1, 2, 2 * w, D) @ k.float().transpose(-1, -2)).reshape(1, 4, w, S) * D ** -0.5
        rp = torch.arange(S - w, S)
        yw = yw.masked_fill(torch.arange(S)[None, :] > rp[:, None], -math.inf)
        pw = torch.softmax(yw, -1)[..., :S - w] * (rp.float()[:, None] if normalize else 1.0)
        f32 = torch.full((1, 2, S), math.inf)
        f32[..., :S - w] = pw.sum(2).reshape(1, 2, 2, S - w).sum(2) / (2 * w)
        ref = torch.full((1, 2, S), math.inf, dtype=torch.float64)
        ref[..., :S - w] = scores64(k, q, w, normalize)
        inside(f32, ref, finch_bound64(k, q, w, normalize), f"finch n{normalize}")
    tova = (r.last(), None, 0.0, 0, False)
    inside(O.expected_attention_scores_fp32(k, r.v, *tova), ea_ref64(k, r.v, *tova), ea_bound64(k, r.v, *tova), "tova")
    for regime in ("mean", "variance"):
        mu, cov = r.ea_stats(regime)
        inside(O.expected_attention_scores_fp32(k, r.v, mu, cov, 0.0, 4, True), ea_ref64(k, r.v, mu, cov, 0.0, 4, True),
               ea_bound64(k, r.v, mu, cov, 0.0, 4, True), f"ea {regime}")


# ---------------------------------------------------------------------------------------------------
# 3. the sweep: every scorer, both dtypes, head_dim 64 / 128, the group sizes of the instantiation sweeps
#    (SnapKV NQP 128 / 256 / 512, ExpectedAttention GR 1 / 2 / 4 with a short and a second unit, ObservedAttention and
#    Finch G 1-8), the generator grid spread over them
# ---------------------------------------------------------------------------------------------------
GRID = [(0, 0, 1.5), (10, 0, 1.5), (25, 8, 1.5), (0, 30, 4), (0, 0, 12), (25, 30, 12), (10, 8, 4)]
SIZES = [1000, 4097, 8192, 32768]
SCORERS = {
    "snapkv": [(1, 64), (3, 50), (7, 64)],            # (G, window): NQP 128, 256, 512
    "ea": [(1, 0), (2, 0), (3, 0), (4, 0), (8, 0)],
    "tova": [(1, 0), (4, 0)],
    "observed": [(1, 0), (2, 0), (3, 0), (4, 0), (5, 0), (8, 0)],
    "noncausal": [(1, 0), (4, 0)],
    "finch": [(1, 33), (2, 64), (3, 100), (4, 64), (8, 17)],
}
CASES = []
for _name_s, _groups in SCORERS.items():
    for _dt in (BF16, FP16):
        for _D in (64, 128):
            for _G, _w in _groups:
                _i = len(CASES)
                _S = SIZES[_i % len(SIZES)]
                if _name_s in ("observed", "noncausal"):
                    _S = min(_S, 8192)        # their float64 references are quadratic in S
                CASES.append((_name_s, _dt, _D, _G, _w, _S, *GRID[(3 * _i) % len(GRID)]))
CASES += [(n, BF16, 128, 4, w, 131072, 25, 30, 4) for n, w in (("snapkv", 64), ("ea", 0), ("tova", 0), ("finch", 64),
                                                               ("noncausal", 0), ("observed", 0))]


def _id(c):
    n, dt, D, G, w, S, sink, massive, peak = c
    return f"{n}-{_name(dt)}-d{D}-g{G}-w{w}-s{S}-sink{sink}-m{massive}-p{peak}"


def run_case(name, r: RealShaped, dtype, D, G, w, S, what, variant=0):
    """score and compress of one problem against float64 and its E_s; returns (scores, ref)"""
    nat = _native()
    k, v = r.k, r.v
    n_kept = max(1, O.kept_count(S, 0.5))
    if name == "snapkv":
        q = r.window(w)
        sc = nat.snapkv_score(k, q, w, 5)
        ref, E, forced = snap_ref64(q, k, w, 5), snap_bound64(k, q, w, 5), _forced_tail(S, w)
        assert_real(sc, ref, E, forced, what, ftz=True)
        out = nat.snapkv_compress(k, v, q, w, 5, n_kept, return_indices=True, return_scores=True)
    elif name in ("ea", "tova"):
        if name == "ea":
            mu, cov = r.ea_stats("variance" if variant % 2 else "mean")
            args = (mu, cov, 1e-2, 4, True)
        else:
            args = (r.last(), None, 0.0, 0, False)
        sc = nat.expected_attention_score(k, v, *args)
        ref, E = ea_ref64(k, v, *args), ea_bound64(k, v, *args)
        assert_real(sc, ref, E, _forced_head(S, args[3]), what)
        out = nat.expected_attention_compress(k, v, *args, n_kept, return_indices=True, return_scores=True)
    elif name == "observed":
        q = r.q if S <= 8192 else r.q[:, :, -2048:].contiguous()
        sc = nat.observed_attention_score(k, q, D ** -0.5)
        ref, E = oa_ref64(k, q, D ** -0.5), oa_bound64(k, q, D ** -0.5)
        assert_real(sc, ref, E, torch.zeros(S, dtype=torch.bool), what, ftz=True)
        out = nat.observed_attention_compress(k, v, q, D ** -0.5, n_kept, return_indices=True, return_scores=True)
    elif name == "noncausal":
        cs = 128 if variant % 2 else 256  # both instantiations of <T, D, CC>
        sc = nat.non_causal_attention_score(k, v, r.q, cs)
        ref, E = nca_ref(k, v, r.q, cs)
        assert_real(sc, ref, E, torch.zeros(S, dtype=torch.bool), what, bias=False, absolute=True)
        out = nat.non_causal_attention_compress(k, v, r.q, cs, n_kept, return_indices=True, return_scores=True)
    else:  # finch
        normalize = variant % 2 == 0
        q = r.window(w)
        sc = nat.finch_score(k, q, w, normalize)
        ref = torch.full(sc.shape, math.inf, dtype=torch.float64, device=DEV)
        ref[..., :S - w] = scores64(k, q, w, normalize)
        assert_real(sc, ref, finch_bound64(k, q, w, normalize), _forced_tail(S, w), what, ftz=True)
        # Finch's compress keeps per chunk; unchunked it is the plain top-k of its scores with the window forced
        out = nat.finch_compress(k, v, q, w, 0.5, None, normalize, None, True, True)
        n_kept = out[2].shape[-1]
    k_out, v_out, idx, sc2 = out
    assert torch.equal(sc2, sc), f"{what}: compress scores differ from the score path"
    assert_compress(k, v, k_out, v_out, idx, sc2, n_kept)
    return sc, ref


@gpu
@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_real_shaped_sweep(case):
    name, dtype, D, G, w, S, sink, massive, peak = case
    i = CASES.index(case)
    r = real_shaped(1, 2 if S < 131072 else 1, G, S, D, dtype, 1000 + i, sink=sink, massive=massive, peak=peak)
    run_case(name, r, dtype, D, G, w, S, _id(case), variant=i)


# ---------------------------------------------------------------------------------------------------
# 4. exact planted cases
# ---------------------------------------------------------------------------------------------------
def _plant(k, qrows, s_star, margin=120.0):
    """k with key s_star along the mean of qrows [B, H, n, D] (one kv head each), so that its scaled logit beats every
    other key's by `margin` for every row: every other exp2 / __expf underflows to +0 (ftz). Rows in blocks."""
    B, H, S, D = k.shape
    k = k.clone()
    blk = max(1, (1 << 24) // S)
    for b in range(B):
        for h in range(H):
            q = qrows[b, h]
            qbar = q.double().mean(0)
            qhat = qbar / qbar.norm()
            kk = k[b, h].double()
            others = max(float((q[i:i + blk].double() @ kk.T).amax()) for i in range(0, q.shape[0], blk))
            low = min(float((q[i:i + blk].double() @ qhat).min()) for i in range(0, q.shape[0], blk))
            k[b, h, s_star] = ((others + margin * math.sqrt(D) + 1.0) / low * qhat).to(k.dtype)
            kk = k[b, h].double()
            for i in range(0, q.shape[0], blk):
                y = q[i:i + blk].double() @ kk.T
                rest = torch.cat((y[:, :s_star], y[:, s_star + 1:]), -1)
                assert float((y[:, s_star] - rest.amax(-1)).min()) / math.sqrt(D) >= margin - 1
    return k


def _only_one(sc, s_star, forced, want, what, ulp: bool = False):
    """sc[..., s_star] is `want` (bitwise, or within 1 ulp), every other non-forced score +0 (no NaN, no -0)"""
    got = sc[..., s_star]
    if ulp:
        assert (ulp16_diff(got, torch.full_like(got, want)) <= 1).all(), f"{what}: {got.flatten().tolist()} vs {want}"
    else:
        assert (got == want).all(), f"{what}: {got.flatten().tolist()} vs {want}"
    rest = torch.ones(sc.shape[-1], dtype=torch.bool, device=sc.device)
    rest[s_star] = False
    rest &= ~forced.to(sc.device)
    assert (sc[..., rest].view(torch.int16) == 0).all(), f"{what}: a non-dominant score is not +0"


DOM_S, DOM_W = 20000, 64
DOMINANT = [(dt, where) for dt in (BF16, FP16) for where in ("first", "last", "part", "inside_part")]


def dominant_positions(R: int, G: int, S: int, w: int, sm: int):
    """{placement: (SnapKV / Finch / ObservedAttention key, ExpectedAttention key)}. "part": the first key of a
    persistent CTA's part (SnapKV: launch_snap_t's row split, equal in both passes; ExpectedAttention: the second CTA
    of the first unit); "inside_part": the first key of the next tile, strictly inside that part."""
    cpr, _, _ = snap_parts(R, S, w, sm)
    per1, per2 = -(-((S + 127) // 128) // cpr), -(-((S - w + 127) // 128) // cpr)
    assert per1 == per2 >= 2, "the SnapKV parts hold one tile: no tile start inside a part"
    n_tp, _, ranges, spans = ea_schedule(R, G, S)
    first, count = spans[0]
    lo, hi = ranges[first + 1]
    assert count >= 2 and hi - lo >= 2 and lo < n_tp, "the ExpectedAttention parts hold one tile"
    return {"first": (0, 0), "last": (S - w - 1, S - 1), "part": (per2 * 128, lo * 128),
            "inside_part": ((per2 + 1) * 128, (lo + 1) * 128)}


@gpu
@pytest.mark.parametrize("dtype,where", DOMINANT, ids=[f"{_name(d)}-{w}" for d, w in DOMINANT])
def test_one_dominating_key(dtype, where):
    nat = _native()
    B, H, G, S, D, w = 1, 2, 4, DOM_S, 128, DOM_W
    r = real_shaped(B, H, G, S, D, dtype, 77, peak=1.5)
    pos, pos_ea = dominant_positions(B * H, G, S, w, GS._sm_count())[where]
    assert pos < S - w
    # SnapKV / Finch (window rows see keys < S - w), ExpectedAttention (mu rows), ObservedAttention (rows from pos)
    k = _plant(r.k, r.window(w).reshape(B, H, G * w, D), pos)
    f_tail = _forced_tail(S, w)
    sc = nat.snapkv_score(k, r.window(w), w, 1)
    _only_one(sc, pos, f_tail, 1.0, f"snapkv {where}")
    for normalize in (False, True):
        sc = nat.finch_score(k, r.window(w), w, normalize)
        want = (S - w + (w - 1) / 2) if normalize else 1.0
        _only_one(sc, pos, f_tail, want, f"finch {where} n{normalize}", ulp=normalize)
    n_sink = 0 if pos_ea == 0 else 4
    mu = r.last()
    k_ea = _plant(r.k, mu.reshape(B, H, G, D), pos_ea)
    sc = nat.expected_attention_score(k_ea, r.v, mu, None, 0.0, n_sink, False)
    _only_one(sc, pos_ea, _forced_head(S, n_sink), 1.0, f"tova {where}")
    mu_c, cov = r.ea_stats("mean")
    k_ea = _plant(r.k, mu_c.reshape(B, H, G, D), pos_ea, margin=240.0)  # the covariance term adds at most ~100
    ref = ea_ref64(k_ea, r.v, mu_c, cov, 0.0, n_sink, False)
    assert float(ref[..., pos_ea].min()) == 1.0, "the planted key does not take all the mass in float64"
    sc = nat.expected_attention_score(k_ea, r.v, mu_c, cov, 0.0, n_sink, False)
    _only_one(sc, pos_ea, _forced_head(S, n_sink), 1.0, f"ea {where}")
    n_q = S - pos
    qo = r.q[:, :, pos:].contiguous()
    k_o = _plant(r.k, qo.reshape(B, H, G * n_q, D), pos)
    sc = nat.observed_attention_score(k_o, qo, D ** -0.5)
    want = float(n_q / float(torch.tensor(float(n_q)).to(dtype)))
    _only_one(sc, pos, torch.zeros(S, dtype=torch.bool), want, f"observed {where}", ulp=True)


NC_DOMINANT = [(dt, cs) for dt in (BF16, FP16) for cs in (128, 256)]


@gpu
@pytest.mark.parametrize("dtype,cs", NC_DOMINANT, ids=[f"{_name(d)}-cs{c}" for d, c in NC_DOMINANT])
def test_one_dominating_key_per_noncausal_chunk(dtype, cs):
    """NonCausalAttention: the first key of every chunk takes all of its chunk's queries, so x = cs ||v|| there and
    exactly 0 elsewhere (all other exps flush). Its output is a z-score of the pooled x, so the other scores are not 0:
    every position whose pooled window holds no planted key scores -mean / std, bitwise the same, and every score is
    within 1 ulp of the z-score of that closed-form x."""
    nat = _native()
    B, H, G, D = 1, 2, 2, 128
    S = 8 * cs
    r = real_shaped(B, H, G, S, D, dtype, 88, peak=1.5)
    k = r.k
    for c0 in range(0, S, cs):
        k = _plant(k, r.q[:, :, c0:c0 + cs].reshape(B, H, G * cs, D), c0)
    sc = nat.non_causal_attention_score(k, r.v, r.q, cs)
    starts = torch.zeros(S, dtype=torch.bool, device=DEV)
    starts[::cs] = True
    x = torch.where(starts, cs * r.v.double().norm(dim=-1), 0.0)
    z = NB.zscore64(x)
    assert (ulp16_diff(sc, z.to(dtype)) <= 1).all(), f"cs{cs}: beyond 1 ulp of the closed form"
    near = F.max_pool1d(starts.double()[None], 3, 1, 1)[0] > 0
    flat = sc[..., ~near]
    assert (flat.view(torch.int16) == flat.reshape(-1)[0].view(torch.int16)).all(), "the plateau is not one value"
    n_kept = O.kept_count(S, 0.5)
    k_out, v_out, idx, sc2 = nat.non_causal_attention_compress(k, r.v, r.q, cs, n_kept, return_indices=True,
                                                               return_scores=True)
    assert torch.equal(sc2, sc)
    assert_compress(k, r.v, k_out, v_out, idx, sc2, n_kept)


IDENTICAL = [(dt, D) for dt in (BF16, FP16) for D in (64, 128)]


@gpu
@pytest.mark.parametrize("dtype,D", IDENTICAL, ids=[f"{_name(d)}-d{D}" for d, D in IDENTICAL])
def test_identical_keys(dtype, D):
    """Every key (and value) row equal: every softmax is uniform over its visible keys. Each score is within 1 ulp of
    its float64 closed form, and the scores that closed form makes equal are bitwise equal."""
    nat = _native()
    B, H, G, S, w, ksz, n_sink, eps = 1, 2, 4, 3000, 64, 5, 4, 1e-2
    r = real_shaped(B, H, G, S, D, dtype, 99, peak=1.5)
    k = r.k[:, :, 1:2].expand(B, H, S, D).contiguous()
    v = r.v[:, :, 5:6].expand(B, H, S, D).contiguous()
    q = r.window(w)
    n = S - w
    inv = 1.0 / torch.arange(S - w + 1, S + 1, dtype=torch.float64)  # row i sees S - w + i + 1 keys

    def check(got, want, what):
        want = want.to(DEV)
        assert (ulp16_diff(got, want.to(dtype).expand_as(got)) <= 1).all(), f"{what}: beyond 1 ulp of the closed form"

    def same(x, what):
        assert (x.view(torch.int16) == x.reshape(-1)[0].view(torch.int16)).all(), f"{what}: not bitwise equal"

    # SnapKV: the window mean of the uniform rows, then the box filter, which sees fewer of them at both edges
    c = float(inv.sum() / w)
    cnt = F.avg_pool1d(torch.ones(1, 1, n, dtype=torch.float64), ksz, 1, ksz // 2, count_include_pad=True)[0, 0] * ksz
    sc = nat.snapkv_score(k, q, w, ksz)
    check(sc[..., :n], c * cnt / ksz, "snapkv")
    same(sc[..., ksz // 2:n - ksz // 2], "snapkv interior")
    # Finch: the same window mean, without (1 / (w)) sum_i 1 / (S - w + i + 1) or with the position weights
    for normalize in (False, True):
        want = float((inv * (torch.arange(S - w, S, dtype=torch.float64) if normalize else 1.0)).sum() / w)
        sc = nat.finch_score(k, q, w, normalize)
        check(sc[..., :n], torch.tensor(want), f"finch n{normalize}")
        same(sc[..., :n], f"finch n{normalize}")
    # ExpectedAttention: 1 / (S - n_sink), plus eps, times ||v||
    vn = v[0, :, 0].double().norm(dim=-1).cpu()
    want = (1.0 / (S - n_sink) + float(torch.tensor(eps, dtype=torch.float32))) * vn
    for cov in (True, False):
        mu, c_ = r.ea_stats("mean")
        sc = nat.expected_attention_score(k, v, mu, c_ if cov else None, eps, n_sink, True)
        check(sc[..., n_sink:], want[None, :, None], f"ea cov={cov}")
        for h in range(H):
            same(sc[:, h, n_sink:], f"ea cov={cov} head {h}")
    # ObservedAttention: key s is seen by the rows at s .. S - 1, row p uniform over p + 1 keys; / (S - s) in the dtype
    harm = torch.flip(torch.cumsum(torch.flip(1.0 / torch.arange(1, S + 1, dtype=torch.float64), [0]), 0), [0])
    div = torch.arange(S, 0, -1).to(dtype).double()
    sc = nat.observed_attention_score(k, r.q, D ** -0.5)
    check(sc, harm / div, "observed")


def _huge(B, H, G, S, D, w, dtype, seed, amp):
    """keys amp (1 + 0.05 N) s_i and queries -amp (1 + 0.05 N) s_i (s a fixed sign pattern): every raw logit about
    -amp^2 D; the second half of the query heads flipped to +. Masked (causal) keys would dominate a finite stand-in."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    s = torch.randint(0, 2, (D,), generator=g, device=DEV).double() * 2 - 1
    k = amp * (1 + 0.05 * torch.randn(B, H, S, D, generator=g, device=DEV, dtype=torch.float64)) * s
    q = -amp * (1 + 0.05 * torch.randn(B, H * G, S, D, generator=g, device=DEV, dtype=torch.float64)) * s
    q[:, H * G // 2:] *= -1
    v = torch.randn(B, H, S, D, generator=g, device=DEV)
    return RealShaped(k.to(dtype), v.to(dtype), q.to(dtype))


HUGE = [(dt, D) for dt in (BF16, FP16) for D in (64, 128)]


@gpu
@pytest.mark.parametrize("dtype,D", HUGE, ids=[f"{_name(d)}-d{D}" for d, D in HUGE])
def test_huge_raw_logits_of_both_signs(dtype, D):
    """|q.k| of 1e4: window and causal rows whose every valid logit is below -1e4 while later keys are masked"""
    S, G, w = 1500, 2, 64
    amp = 13.0 if D == 64 else 9.0
    r = _huge(1, 2, G, S, D, w, dtype, 5 + D, amp)
    y = r.q[0, 0, -w:].double() @ r.k[0, 0].double().T
    assert float(y.max()) < -1e4 and float(y.min()) > -2e4
    for name in ("snapkv", "finch", "observed", "ea", "tova", "noncausal"):
        run_case(name, r, dtype, D, G, w, S, f"huge {name} {_name(dtype)} d{D}", variant=1 if name == "ea" else 0)


@gpu
def test_selection_on_a_plateau_of_zeros():
    """Peaked fp16 rows: thousands of +0 scores, n_kept inside the plateau. The kept set is the lowest-index ties of
    the kernel's scores, and holds every position whose float64 score is a normal fp16 number."""
    nat = _native()
    S, D, G, w = 8192, 128, 4, 64
    r = real_shaped(1, 2, G, S, D, FP16, 9, peak=12)
    q = r.window(w)
    for name in ("snapkv", "finch"):
        if name == "snapkv":
            sc = nat.snapkv_score(r.k, q, w, 1)
            ref = snap_ref64(q, r.k, w, 1)
        else:
            sc = nat.finch_score(r.k, q, w, False)
            ref = torch.full(sc.shape, math.inf, dtype=torch.float64, device=DEV)
            ref[..., :S - w] = scores64(r.k, q, w, False)
        zeros = (sc[..., :S - w] == 0).sum(-1)
        assert int(zeros.min()) >= 2000, f"{name}: the plateau holds {zeros.tolist()} positions"
        n_kept = int((sc != 0).sum(-1).max()) + 700
        k_out, v_out, idx = nat.scores_compress(sc, r.k, r.v, n_kept, return_indices=True)
        assert_compress(r.k, r.v, k_out, v_out, idx, sc, n_kept)
        above = ref >= torch.finfo(FP16).tiny
        kept = torch.zeros_like(above).scatter_(-1, idx.long(), True)
        assert (kept | ~above).all(), f"{name}: a position above the plateau is not kept"


@gpu
def test_ea_sentinel_overflow_keeps_the_sinks():
    """bf16 value norms >= 256: the call's largest score, about 1000, has an ulp of 4, so the sentinel round(max + 1)
    equals max and the forced sinks only tie the best position of the head that holds it. They are still kept: ties go
    to the lowest position, and the sinks are positions 0 .. n_sink - 1."""
    nat = _native()
    B, H, G, S, D, n_sink = 1, 2, 4, 3000, 128, 4
    r = real_shaped(B, H, G, S, D, BF16, 31, peak=1.5)
    mu = r.last()
    s_star = 1000
    k = _plant(r.k, mu.reshape(B, H, G, D), s_star)
    v = r.v.double()
    norms = 300.0 + 700.0 * torch.rand(B, H, S, 1, generator=torch.Generator(DEV).manual_seed(3), device=DEV,
                                       dtype=torch.float64)
    v = (v / v.norm(dim=-1, keepdim=True) * norms).to(BF16)
    v[:, :, s_star] = (v[:, :, s_star].double() / v[:, :, s_star].double().norm(dim=-1, keepdim=True) * 1000).to(BF16)
    sc = nat.expected_attention_score(k, v, mu, None, 1e-2, n_sink, True)
    top = sc[..., n_sink:].amax()  # the sentinel is round(max + 1) over the whole call
    info = f"max {float(top)}, at s_star {sc[..., s_star].tolist()}, sinks {sc[..., :n_sink].tolist()}"
    assert (top.float() + 1).to(BF16) == top, info
    assert (sc[..., :n_sink] == top).all() and (sc[..., s_star] == sc[..., n_sink:].amax(-1)).all(), info
    assert (sc[..., s_star] == top).any(), info
    n_kept = n_sink + 1
    k_out, v_out, idx, _ = nat.expected_attention_compress(k, v, mu, None, 1e-2, n_sink, True, n_kept,
                                                           return_indices=True)
    want = torch.tensor(list(range(n_sink)) + [s_star], device=DEV).expand(B, H, n_kept)
    assert torch.equal(idx.long(), want)
    assert_compress(k, v, k_out, v_out, idx, sc, n_kept)
