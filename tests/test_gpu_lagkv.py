"""LagKV on the GPU: the sm_90a kernel (csrc/lagkv.cu) against a float64 evaluation of its definition
(include/kvpress_b200.h, kvp_lagkv_score), from the same 16-bit inputs, on the device (tests/lagkv_backend.py).

Positions outside the scored partitions (the sinks, the last partition, the remainder, and the whole short cache) are
fp32 quotients rounded once: they must equal the float64 backend bitwise. Inside the scored partitions, with c64 the
float64 combined score, u = 2^-24 the fp32 unit roundoff and ulp the spacing of the cache dtype:
1. Cross scores: each is within 1 ulp of c64 rounded once, or |c - c64| <= ulp / 2 + E_s, where E_s bounds the kernel's
   fp32 error before the one rounding. The E_s arm may decide at most 1 % of a case's positions. No row bias: over a
   row's positions (at least 500), the mean of (c - c64) / ulp is within 8 / sqrt(12 n). NaN exactly where c64 is NaN.
2. Ranks: each partition's outputs are exactly the multiset {round(r / L) : r = 0 ... L-1}. Each output lies between
   round(r_lo / L) and round(r_hi / L), the float64 ranks when pairs with |c64_t - c64_s| <= E_s + E_t may go either
   way. At most 1 % of positions differ from round(r64 / L). NaN partitions rank in position order exactly.

E_s, derived from the kernel's operations (first order; the final factor 1.01 covers the second-order terms):
- x = (k - lo) / (hi - lo): two fp32 subtractions and one division of exact 16-bit inputs, |dx_d| <= 3 u |x_d|.
- mean = (sum of D x_d) / D, summed in fp32 (8 per lane, then a butterfly) and divided:
  |d mean| <= (D + 4) u sum_d |x_d| / D.
- e_d = x_d - mean: |d e_d| <= 3 u |x_d| + |d mean| + u |e_d|.
- q = sum_d e_d^2 (fmas, fp32): |dq| <= sum_d (2 |e_d| |d e_d| + |d e_d|^2) + (D + 1) u q; var = q / (D - 1) adds u var:
  dvar = |dq| / (D - 1) + u var.
- sigma = sqrtf(var): |d sigma| <= 2 dvar / (sigma + sqrt(dvar)) + u sigma =: E_sigma (valid for any dvar, also
  near sigma = 0).
- a = expf(sigma - m) / Z: the exponent carries E_sigma(s) + max_t E_sigma(t) (m is the computed maximum) + the
  subtraction's u |sigma - m|, expf adds 2 ulp (4 u): de_s. Z sums L such terms in fp32: dZ <= max_t de_t + L u. The
  division adds u: |da_s| <= a_s (de_s + dZ + u).
- c = (a_k + a_v) * 0.5: E_s = 1.01 ((|da_k| + |da_v|) / 2 + u c).
"""
import math

import pytest
import torch
from transformers import DynamicCache

from oracle import press_oracle as O
from tests import lagkv_backend as LB
from tests.conftest import ulp16_diff
from tests.gpu_support import (assert_compress, gpu_ids, lagkv_inputs, LANES_PER_ROW, lanes_per_row, _masked, _name,
                               _native, _prefill, same16, _shared, tiny_gpu_llama, ulp_at)

gpu = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24
LAG_MAX = 1024


# --------------------------------------------------------------------------------------------------
# the bounds of the module docstring
# --------------------------------------------------------------------------------------------------
def sigma_bound(x16, n_sink: int, L: int):
    """(sigma64, E_sigma) of every scored row, [B, H, P - 1, L]."""
    B, H, S, D = x16.shape
    P = (S - n_sink) // L
    t = x16[:, :, n_sink:n_sink + P * L].double().reshape(B, H, P, L, D)
    lo = t[:, :, 1:].amin(dim=-2, keepdim=True)
    hi = t[:, :, 1:].amax(dim=-2, keepdim=True)
    x = (t[:, :, :-1] - lo) / (hi - lo)
    del t
    mean = x.mean(dim=-1, keepdim=True)
    dmean = (D + 4) * U * x.abs().sum(dim=-1, keepdim=True) / D
    e = x - mean
    de = 3 * U * x.abs() + dmean + U * e.abs()
    del x
    q = (e * e).sum(dim=-1)
    dq = (2 * e.abs() * de + de * de).sum(dim=-1) + (D + 1) * U * q
    var = q / (D - 1)
    sigma = var.sqrt()
    dvar = dq / (D - 1) + U * var
    return sigma, 2 * dvar / (sigma + dvar.sqrt()) + U * sigma


def combined_bound(keys, values, n_sink: int, L: int):
    """(c64, E_s) of every scored position, [B, H, P - 1, L]."""
    def softmax_bound(x16):
        s, E = sigma_bound(x16, n_sink, L)
        m = s.amax(dim=-1, keepdim=True)
        de = E + E.amax(dim=-1, keepdim=True) + U * (s - m).abs() + 4 * U
        a = (s - m).exp()
        a = a / a.sum(dim=-1, keepdim=True)
        dz = de.amax(dim=-1, keepdim=True) + L * U
        return a, a * (de + dz + U)

    ak, dak = softmax_bound(keys)
    av, dav = softmax_bound(values)
    c = (ak + av) / 2
    return c, 1.01 * ((dak + dav) / 2 + U * c)


def rank_bounds(c64, E):
    """(r_lo, r_hi): the float64 ranks when pairs within E_s + E_t may go either way, per block of partitions."""
    shape = c64.shape
    L = shape[-1]
    c, e = c64.reshape(-1, L), E.reshape(-1, L)
    lo = torch.empty_like(c, dtype=torch.int64)
    hi = torch.empty_like(c, dtype=torch.int64)
    step = max(1, (1 << 24) // (L * L))
    for i in range(0, c.shape[0], step):
        cs, es = c[i:i + step, :, None], e[i:i + step, :, None]
        ct, et = c[i:i + step, None, :], e[i:i + step, None, :]
        lo[i:i + step] = (ct + et < cs - es).sum(dim=-1)
        hi[i:i + step] = (ct - et <= cs + es).sum(dim=-1) - 1
    return lo.view(shape), hi.view(shape)


def check(k, v, n_sink: int, L: int, cross: bool, sc, what: str, bias: bool = True) -> dict:
    """Both bars of the module docstring for the scores `sc` of (k, v)."""
    B, H, S, D = k.shape
    dtype = sc.dtype
    want = LB.lagkv_score(k, v, n_sink, L, cross)
    if LB.is_short(S, n_sink, L):
        assert same16(sc, want), f"{what}: short cache differs"
        return {}
    P = (S - n_sink) // L
    a, b = n_sink, n_sink + (P - 1) * L
    assert torch.equal(sc[..., :a], want[..., :a]) and torch.equal(sc[..., b:], want[..., b:]), f"{what}: constants"
    got = sc[..., a:b].reshape(B, H, P - 1, L)
    c64, E = combined_bound(k, v, n_sink, L)
    nan = torch.isnan(c64)
    part_nan = nan.any(dim=-1)
    assert torch.equal(nan, part_nan[..., None].expand_as(nan)), "a NaN c64 makes its whole partition NaN"
    if cross:
        assert torch.equal(torch.isnan(got), nan), f"{what}: NaN positions differ"
        g, z, e = got[~nan], c64[~nan], E[~nan]
        if g.numel() == 0:
            return {"nan_partitions": int(part_nan.sum())}
        d = ulp16_diff(g, z.to(dtype))
        near = (g.double() - z).abs() <= ulp_at(z, dtype) / 2 + e
        ok = (d <= 1) | near
        assert ok.all(), f"{what}: {int((~ok).sum())} positions beyond both bars (max {int(d.max())} ulp)"
        e_arm = int(((d > 1) & near).sum())
        assert e_arm <= max(1, d.numel() // 100), f"{what}: the E_s arm decides {e_arm} of {d.numel()} positions"
        if bias:
            rel = ((got.double() - c64) / ulp_at(c64, dtype)).reshape(B * H, -1)
            for r, m in zip(rel, (~nan).reshape(B * H, -1)):
                n = int(m.sum())
                if n >= 500:
                    assert abs(float(r[m].mean())) <= 8 / math.sqrt(12 * n), f"{what}: row bias {float(r[m].mean())}"
        return {"max_ulp": int(d.max()), "e_arm": e_arm}
    # ranks: each partition is the multiset {round(r / L)}
    levels = (torch.arange(L, device=sc.device, dtype=torch.float32) / L).to(dtype)
    assert torch.equal(got.sort(dim=-1).values, levels.expand_as(got)), f"{what}: not a permutation of the ranks"
    r64 = LB.ranks(c64)
    exact = (r64.to(torch.float32) / L).to(dtype)
    assert torch.equal(got[part_nan], exact[part_nan]), f"{what}: NaN partitions must rank in position order"
    r_lo, r_hi = rank_bounds(c64, E)
    lo_v = (r_lo.to(torch.float32) / L).to(dtype).float()
    hi_v = (r_hi.to(torch.float32) / L).to(dtype).float()
    inside = (got.float() >= lo_v) & (got.float() <= hi_v)
    assert inside[~part_nan].all(), f"{what}: {int((~inside[~part_nan]).sum())} ranks outside their float64 range"
    differ = int((got != exact).sum())
    assert differ <= got.numel() // 100, f"{what}: {differ} of {got.numel()} ranks differ from float64"
    return {"rank_differ": differ}


def run(k, v, n_sink, L, cross, what, n_kept=None, bias=True):
    """score and compress of one problem, checked; returns the scores."""
    nat = _native()
    S = k.shape[2]
    sc = nat.lagkv_score(k, v, n_sink, L, cross)
    check(k, v, n_sink, L, cross, sc, what, bias=bias)
    assert same16(nat.lagkv_score(k, v, n_sink, L, cross), sc), f"{what}: two calls differ"
    n_kept = max(1, O.kept_count(S, 0.5)) if n_kept is None else n_kept
    k_out, v_out, idx, sc2 = nat.lagkv_compress(k, v, n_sink, L, cross, n_kept, return_indices=True,
                                                return_scores=True)
    assert same16(sc2, sc), f"{what}: compress scores differ from the score call"
    assert_compress(k, v, k_out, v_out, idx, sc2, n_kept)
    return sc


# --------------------------------------------------------------------------------------------------
# every instantiation, every lag size, the boundaries of S
# --------------------------------------------------------------------------------------------------
HEAD_DIMS = (8, 16, 40, 64, 72, 96, 128, 200, 256)
SWEEP = [(dt, D, cross) for dt in (torch.bfloat16, torch.float16) for D in HEAD_DIMS for cross in (False, True)]


def test_sweep_reaches_every_lanes_per_row_instantiation():
    """CPU: the lanes-per-row instantiations of lagkv.cu, per dtype, are all reached by SWEEP."""
    reached = {(_name(dt), lanes_per_row(D), cross) for dt, D, cross in SWEEP}
    assert reached == {(n, lpr, cross) for n in ("bf16", "fp16") for lpr in LANES_PER_ROW for cross in (False, True)}
    assert {lanes_per_row(D) for D in HEAD_DIMS if D // 8 < lanes_per_row(D)} == set(LANES_PER_ROW)  # idle lanes


@gpu
@pytest.mark.parametrize("dtype,D,cross", SWEEP, ids=[f"{_name(dt)}-d{D}-{'cross' if c else 'rank'}"
                                                       for dt, D, c in SWEEP])
def test_instantiations(dtype, D, cross):
    k, v = lagkv_inputs(1, 2, 4 + 12 * 128 + 37, D, dtype, seed=D + 7 * cross)
    run(k, v, 4, 128, cross, f"lagkv {_name(dtype)} d{D} cross={cross}")


LAGS = (1, 2, 7, 100, 128, 256, 1000, LAG_MAX)


@gpu
@pytest.mark.parametrize("cross", [False, True], ids=["rank", "cross"])
@pytest.mark.parametrize("L", LAGS)
def test_lag_sizes(L, cross):
    dtype = (torch.bfloat16, torch.float16)[LAGS.index(L) % 2]
    n_parts = 6 if L >= 100 else 40
    S = 4 + n_parts * L + L // 3
    k, v = lagkv_inputs(2, 2, S, 128, dtype, seed=L)
    sc = run(k, v, 4, L, cross, f"lagkv L{L} cross={cross}")
    if L == 1:  # one-row reference partitions: every scored partition is NaN
        scored = sc[..., 4:4 + (n_parts - 1)]
        assert (torch.isnan(scored).all() if cross else (scored == 0).all())


def _edges():
    out = set()
    for n_sink in (0, 4):
        for L in (16, 128):
            for base in (n_sink + 2 * L, n_sink + 3 * L, n_sink + 7 * L):
                out.update((S, n_sink, L) for S in (base - 1, base, base + 1))
    out.update({(1, 4, 16), (1, 0, 16), (4, 4, 16), (5, 4, 16), (40, 40, 16), (40, 64, 16), (300, 299, 16)})
    return sorted(out)


EDGES = _edges()


@gpu
@pytest.mark.parametrize("cross", [False, True], ids=["rank", "cross"])
@pytest.mark.parametrize("S,n_sink,L", EDGES, ids=[f"s{S}-sink{n}-L{L}" for S, n, L in EDGES])
def test_sequence_edges(S, n_sink, L, cross):
    i = EDGES.index((S, n_sink, L))
    dtype, D, _ = SWEEP[(5 * i) % len(SWEEP)]
    k, v = lagkv_inputs(1, 3, S, D, dtype, seed=1000 + i)
    run(k, v, n_sink, L, cross, f"lagkv {_name(dtype)} d{D} S{S} sink{n_sink} L{L}", n_kept=max(1, S // 3),
        bias=False)


@gpu
@pytest.mark.parametrize("cross", [False, True], ids=["rank", "cross"])
@pytest.mark.parametrize("S", [4096, 16384, 32768, 131072])
def test_llama_layer_shape(S, cross):
    """The Llama-3.1-8B layer shape [1, 8, S, 128] bf16 with the reference defaults, up to 128k."""
    k, v = lagkv_inputs(1, 8, S, 128, torch.bfloat16, seed=S % 997)
    run(k, v, 4, 128, cross, f"lagkv llama8b S{S}", n_kept=O.kept_count(S, 0.5))


@gpu
def test_thousands_of_rows_and_a_row_alone():
    """B Hkv = 3000: a row's scores are bitwise those of the same row scored alone."""
    nat = _native()
    k, v = lagkv_inputs(3, 1000, 4 + 9 * 32 + 5, 64, torch.float16, seed=3)
    for cross in (False, True):
        sc = run(k, v, 4, 32, cross, f"lagkv 3000 rows cross={cross}")
        for b, h in ((0, 0), (1, 517), (2, 999)):
            alone = nat.lagkv_score(k[b:b + 1, h:h + 1].contiguous(), v[b:b + 1, h:h + 1].contiguous(), 4, 32, cross)
            assert same16(alone[0, 0], sc[b, h])


# --------------------------------------------------------------------------------------------------
# special cases
# --------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("cross", [False, True], ids=["rank", "cross"])
def test_degenerate_partitions(cross):
    """A constant K channel in partition 3 makes partition 2 NaN (ranks in position order, cross NaN); a zeroed V
    channel everywhere makes every scored partition of that head NaN; an all-equal partition ranks by position."""
    nat = _native()
    L, n_sink = 32, 4
    k, v = lagkv_inputs(1, 3, n_sink + 8 * L + 9, 64, torch.bfloat16, seed=21)
    k[0, 0, n_sink + 3 * L:n_sink + 4 * L, 17] = 0.5
    v[0, 1, :, 40] = 0
    k[0, 2, n_sink + 5 * L:n_sink + 6 * L] = k[0, 2, n_sink + 5 * L]
    v[0, 2, n_sink + 5 * L:n_sink + 6 * L] = v[0, 2, n_sink + 5 * L]
    sc = run(k, v, n_sink, L, cross, f"lagkv degenerate cross={cross}", bias=False)
    ramp = (torch.arange(L, device=DEV, dtype=torch.float32) / L).to(sc.dtype)
    part = sc[0, 0, n_sink + 2 * L:n_sink + 3 * L]
    assert torch.isnan(part).all() if cross else torch.equal(part, ramp)
    head1 = sc[0, 1, n_sink:n_sink + 7 * L]
    assert torch.isnan(head1).all() if cross else torch.equal(head1.view(7, L), ramp.expand(7, L))
    equal = sc[0, 2, n_sink + 5 * L:n_sink + 6 * L]
    assert (equal == equal[0]).all() if cross else torch.equal(equal, ramp)
    # all-zero V: every scored position of every head is NaN or in position order
    zero = nat.lagkv_score(k, torch.zeros_like(v), n_sink, L, cross)[..., n_sink:n_sink + 7 * L]
    assert torch.isnan(zero).all() if cross else torch.equal(zero, ramp.repeat(7).expand_as(zero))


@gpu
@pytest.mark.parametrize("cross", [False, True], ids=["rank", "cross"])
def test_nan_input_propagates_like_torch_min_max(cross):
    """A NaN in K (head 0, partition 4) and in V (head 1, partition 2): the partition holding it and the partition it is
    the reference of are NaN, as torch.min / max carry the NaN into lo / hi."""
    nat = _native()
    L, n_sink = 32, 4
    k, v = lagkv_inputs(1, 2, n_sink + 8 * L + 9, 64, torch.bfloat16, seed=23)
    k[0, 0, n_sink + 4 * L + 5, 11] = float("nan")
    v[0, 1, n_sink + 2 * L + 30, 60] = float("nan")
    sc = nat.lagkv_score(k, v, n_sink, L, cross)
    check(k, v, n_sink, L, cross, sc, f"lagkv NaN input cross={cross}", bias=False)
    assert same16(nat.lagkv_score(k, v, n_sink, L, cross), sc)
    ramp = (torch.arange(L, device=DEV, dtype=torch.float32) / L).to(sc.dtype)
    for h, p in ((0, 4), (1, 2)):
        for c in (p - 1, p):
            part = sc[0, h, n_sink + c * L:n_sink + (c + 1) * L]
            assert torch.isnan(part).all() if cross else torch.equal(part, ramp)
        other = sc[0, h, n_sink + (p + 1) * L:n_sink + (p + 2) * L]
        assert not torch.isnan(other).any()


@gpu
def test_planted_ties_rank_by_position():
    """Duplicate (k, v) rows inside a partition get equal c: they rank in position order, exactly."""
    L, n_sink = 64, 4
    k, v = lagkv_inputs(2, 2, n_sink + 6 * L + 3, 128, torch.bfloat16, seed=5)
    p0 = n_sink + 2 * L
    dup = [p0 + 3, p0 + 10, p0 + 40, p0 + 63]
    k[:, :, dup], v[:, :, dup] = k[:, :, p0 + 20:p0 + 21], v[:, :, p0 + 20:p0 + 21]
    dup = sorted(dup + [p0 + 20])
    sc = run(k, v, n_sink, L, False, "lagkv planted ties", bias=False)
    cross = _native().lagkv_score(k, v, n_sink, L, True)
    assert (cross[..., dup] == cross[..., dup[:1]]).all()
    ranks = (sc[..., dup].float() * L).round()
    assert (ranks[..., 1:] - ranks[..., :-1] == 1).all(), "equal scores must take consecutive ranks in position order"


@gpu
@pytest.mark.parametrize("cross", [False, True], ids=["rank", "cross"])
def test_fp16_near_the_top_of_the_range(cross):
    k, v = lagkv_inputs(1, 2, 4 + 10 * 128, 128, torch.float16, seed=8, scale=1.0)
    k = (k.float() / k.float().abs().amax() * 65000).half()
    v = (v.float() / v.float().abs().amax() * 60000).half()
    assert torch.isfinite(k).all() and torch.isfinite(v).all()
    run(k, v, 4, 128, cross, f"lagkv fp16 top of range cross={cross}")


# --------------------------------------------------------------------------------------------------
# layouts and schedules: bitwise equal to contiguous copies
# --------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("layout", ["strided", "transposed", "slice"])
def test_layouts(layout):
    nat = _native()
    B, H, S, D = 2, 4, 3000, 128
    k, v = lagkv_inputs(B, H, S, D, torch.bfloat16, seed=7)
    if layout == "strided":  # rows of D within rows of D + 64
        kb = torch.zeros((B, H, S, D + 64), dtype=k.dtype, device=DEV)
        vb = torch.zeros_like(kb)
        kb[..., :D], vb[..., :D] = k, v
        k, v = kb[..., :D], vb[..., :D]
    elif layout == "transposed":  # [B, S, H, D] caches viewed as [B, H, S, D]
        k = k.transpose(1, 2).contiguous().transpose(1, 2)
        v = v.transpose(1, 2).contiguous().transpose(1, 2)
    else:  # keys[..., a:b, :], as ChunkPress slices chunks
        k, v = k[..., 8:-4, :], v[..., 8:-4, :]
        assert not k.is_contiguous() and nat._rows_ok(k)
    for cross in (False, True):
        sc = run(k, v, 4, 128, cross, f"lagkv {layout}")
        assert same16(sc, nat.lagkv_score(k.contiguous(), v.contiguous(), 4, 128, cross))


def scoring_items(R: int, n_scored: int, sm: int) -> int:
    """The kernel's segments (csrc/lagkv.cu, launch_lagkv_score): 2 per SM over the rows, at most one per partition."""
    per_row = min(n_scored, max(1, -(-2 * sm // R)))
    seg_len = -(-n_scored // per_row)
    return R * -(-n_scored // seg_len)


@gpu
@pytest.mark.parametrize("regime", ["fewer", "equal", "more"])
def test_schedule_regimes(regime):
    """Scoring items fewer than, equal to and more than the SMs (one row; R = 8 with long segments for 'more')."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    R, n_scored = {"fewer": (1, sm // 2), "equal": (1, sm), "more": (8, 4 * sm + 5)}[regime]
    items = scoring_items(R, n_scored, sm)
    assert (items < sm, items == sm, items > sm)[["fewer", "equal", "more"].index(regime)], (items, sm)
    L = 16
    S = 4 + (n_scored + 1) * L + 3
    k, v = lagkv_inputs(1, R, S, 64, torch.float16, seed=n_scored)
    for cross in (False, True):
        run(k, v, 4, L, cross, f"lagkv schedule {regime} ({items} items, {sm} SMs)")


# --------------------------------------------------------------------------------------------------
# compress: edges of n_kept, determinism, graph replay, workspace check, memory
# --------------------------------------------------------------------------------------------------
@gpu
def test_compress_edges_and_n_kept_zero():
    nat = _native()
    k, v = lagkv_inputs(2, 2, 4 + 5 * 128 + 50, 64, torch.bfloat16, seed=12)
    S = k.shape[2]
    for cross in (False, True):
        for n_kept in (1, S):
            run(k, v, 4, 128, cross, f"lagkv n_kept {n_kept}", n_kept=n_kept)
    p = nat.make_problem(k, v, 0)
    ws = nat._workspace(p, nat.SCORER_LAGKV, k.device)
    outs = [torch.full((2, 2, 0, 64), 3, dtype=k.dtype, device=DEV) for _ in range(2)]
    idx = torch.full((2, 2, 1), -5, dtype=torch.int32, device=DEV)
    scores = torch.full((2, 2, S), 7, dtype=k.dtype, device=DEV)
    lib = nat.load()
    import ctypes
    rc = lib.kvp_lagkv_compress(ctypes.byref(p), k.data_ptr(), v.data_ptr(), 4, 128, 0, outs[0].data_ptr(),
                                outs[1].data_ptr(), ctypes.cast(idx.data_ptr(), ctypes.POINTER(ctypes.c_int32)),
                                scores.data_ptr(), ws.data_ptr(), ws.numel(), nat._stream())
    torch.cuda.synchronize()
    assert rc == 0 and (idx == -5).all() and (scores == 7).all()


@gpu
def test_replays_under_capture_and_workspace_check():
    nat = _native()
    k, v = lagkv_inputs(1, 8, 8000, 128, torch.bfloat16, seed=9)
    eager = nat.lagkv_compress(k, v, 4, 128, False, 4000, True, True)
    again = nat.lagkv_compress(k, v, 4, 128, False, 4000, True, True)
    assert all(same16(a, b) for a, b in zip(eager, again))
    g = nat.capture(lambda: (nat.lagkv_score(k, v, 4, 128, True), *nat.lagkv_compress(k, v, 4, 128, False, 4000,
                                                                                         True, True)))
    out = g.replay()
    torch.cuda.synchronize()
    assert all(same16(a, b) for a, b in zip(out[1:], eager))
    k.copy_(torch.randn_like(k.float()).to(k.dtype))  # inputs updated in place
    v.mul_(-1)
    out = g.replay()
    torch.cuda.synchronize()
    fresh = (nat.lagkv_score(k, v, 4, 128, True), *nat.lagkv_compress(k, v, 4, 128, False, 4000, True, True))
    assert all(same16(a, b) for a, b in zip(out, fresh))
    assert not torch.equal(out[3], eager[2])
    p = nat.make_problem(k, v, 4000)
    nat.workspace_check(p, nat.SCORER_LAGKV, nat._workspace(p, nat.SCORER_LAGKV, k.device))


@gpu
def test_no_intermediate_at_128k():
    """Memory grows by no more than the workspace and the outputs: no cache-sized temporary."""
    nat = _native()
    B, H, S, D = 1, 8, 131072, 128
    k, v = lagkv_inputs(B, H, S, D, torch.bfloat16, seed=10)
    n_kept = S // 2
    p = nat.make_problem(k, v, n_kept)
    ws = nat.workspace_bytes(p, nat.SCORER_LAGKV)
    nat._WS_CACHE.clear()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    out = nat.lagkv_compress(k, v, 4, 128, False, n_kept, True, True)
    torch.cuda.synchronize()
    outputs = sum(t.numel() * t.element_size() for t in out if t is not None)
    grown = torch.cuda.max_memory_allocated() - before
    assert grown <= max(ws, 1 << 20) + outputs + (1 << 16), (grown, ws, outputs)


@gpu
def test_unsupported_lag_and_the_press_fallback():
    """lag_size > 1024 is refused by the kernel; the press scores it with its float32 torch evaluation and compresses
    with the shared selection kernels."""
    from kvpress_b200 import LagKVPress

    nat = _native()
    L = LAG_MAX + 1
    k, v = lagkv_inputs(1, 2, 4 + 4 * L + 11, 64, torch.bfloat16, seed=4)
    with pytest.raises(RuntimeError, match="unsupported shape"):
        nat.lagkv_score(k, v, 4, L, False)
    with pytest.raises(RuntimeError, match="bad argument"):
        nat.lagkv_score(k, v, -1, 128, False)
    for cross in (False, True):
        press = LagKVPress(compression_ratio=0.5, lag_size=L, cross_scoring=cross)
        sc = press.score(None, None, k, v, None, {})
        want = LB.lagkv_score(k, v, 4, L, cross)
        if cross:
            assert (ulp16_diff(sc, want) <= 1).float().mean() >= 0.99 and (ulp16_diff(sc, want) <= 2).all()
        else:
            assert (sc != want).float().mean() <= 0.01
        k_out, v_out = press.compress(None, None, k, v, None, {})
        idx = O.select_lowest_index_ties(sc.cpu(), O.kept_count(k.shape[2], 0.5)).to(DEV)
        assert torch.equal(k_out, O.gather_rows(k, idx)) and torch.equal(v_out, O.gather_rows(v, idx))


# --------------------------------------------------------------------------------------------------
# presses on a GPU tiny Llama, every native call checked against the float64 definition
# --------------------------------------------------------------------------------------------------


@pytest.fixture
def checked(monkeypatch):
    """Wraps native.lagkv_score / lagkv_compress: every call's scores meet the bars, and its selection is canonical."""
    from kvpress_b200 import native

    calls = []
    real_score, real_compress = native.lagkv_score, native.lagkv_compress

    def score(keys, values, n_sink, lag_size, cross):
        sc = real_score(keys, values, n_sink, lag_size, cross)
        check(keys, values, n_sink, lag_size, cross, sc, "press score call", bias=False)
        calls.append(("score", keys.shape[2]))
        return sc

    def compress(keys, values, n_sink, lag_size, cross, n_kept, return_indices=False, return_scores=False):
        k_out, v_out, idx, sc = real_compress(keys, values, n_sink, lag_size, cross, n_kept, True, True)
        check(keys, values, n_sink, lag_size, cross, sc, "press compress call", bias=False)
        assert_compress(keys, values, k_out, v_out, idx, sc, n_kept)
        calls.append(("compress", keys.shape[2]))
        return k_out, v_out, idx if return_indices else None, sc if return_scores else None

    monkeypatch.setattr(native, "lagkv_score", score)
    monkeypatch.setattr(native, "lagkv_compress", compress)
    return calls


def _standin(press_factory, forward, monkeypatch):
    """(model, cache) the same press leaves, run through `forward`, with the float64 stand-ins in place of the
    kernels."""
    with monkeypatch.context() as m:
        LB.install(m)
        model, cache = tiny_gpu_llama(), DynamicCache()
        with press_factory()(model):
            forward(model, cache)
    return model, cache


def _standin_rows(press_factory, ids, monkeypatch):
    """The cache the same press leaves on a prefill of `ids` with the float64 stand-ins."""
    return _standin(press_factory, _prefill(ids), monkeypatch)[1]


@gpu
@pytest.mark.parametrize("cross", [False, True], ids=["rank", "cross"])
def test_press_on_a_tiny_llama(checked, monkeypatch, cross):
    from kvpress_b200 import LagKVPress

    ids = gpu_ids()
    factory = lambda: LagKVPress(compression_ratio=0.5, lag_size=16, cross_scoring=cross)  # noqa: E731
    model, cache = tiny_gpu_llama(), DynamicCache()
    with factory()(model):
        model.model(input_ids=ids, past_key_values=cache)
    assert cache.get_seq_length() == 120 and checked == [("compress", 240)] * 2
    assert _shared(cache, _standin_rows(factory, ids, monkeypatch)) >= 0.97


@gpu
def test_wrapper_presses_on_a_tiny_llama(checked, monkeypatch):
    """AdaKV, KeyRerotation, ChunkPress and DecodingPress over LagKVPress: every native call meets the float64 bars
    (the `checked` fixture), and each press leaves what it leaves with the float64 stand-ins, but for the near-ties at
    its threshold (97 % of the masked positions or kept rows shared)."""
    from kvpress_b200 import AdaKVPress, ChunkPress, DecodingPress, KeyRerotationPress, LagKVPress

    ids = gpu_ids()
    model = tiny_gpu_llama()
    cache = DynamicCache()
    ada = lambda: AdaKVPress(LagKVPress(compression_ratio=0.5, lag_size=16, cross_scoring=True))  # noqa: E731
    with ada()(model):
        _prefill(ids)(model, cache)
    attn = [layer.self_attn for layer in model.model.layers]
    assert cache.get_seq_length() == 240 and all(a.masked_key_indices is not None for a in attn)
    assert checked == [("score", 240)] * 2
    ours, theirs = _masked(model), _masked(_standin(ada, _prefill(ids), monkeypatch)[0])
    for a, b in zip(ours, theirs):
        assert len(a) == len(b) == 2 * 2 * 120 and len(a & b) >= 0.97 * len(a)
    for a in attn:
        a.masked_key_indices = None

    rerotate = lambda: KeyRerotationPress(LagKVPress(compression_ratio=0.5, lag_size=16))  # noqa: E731
    logits = []

    def with_logits(m, c):
        logits.append(m(input_ids=ids, past_key_values=c).logits)

    cache = DynamicCache()
    with rerotate()(model):
        with_logits(model, cache)
    assert cache.get_seq_length() == 120 and torch.isfinite(logits[0].float()).all()
    assert _shared(cache, _standin(rerotate, with_logits, monkeypatch)[1]) >= 0.97

    del checked[:]
    chunk = lambda: ChunkPress(LagKVPress(compression_ratio=0.5, lag_size=16), chunk_length=64)  # noqa: E731
    cache = DynamicCache()
    with chunk()(model):
        _prefill(ids)(model, cache)
    assert cache.get_seq_length() == 120 and checked == ([("score", 64)] * 3 + [("score", 48)]) * 2
    assert _shared(cache, _standin_rows(chunk, ids, monkeypatch)) >= 0.97

    del checked[:]
    decoding = lambda: DecodingPress(LagKVPress(lag_size=16), compression_interval=4, target_size=100)  # noqa: E731

    def decode(m, c):
        m.model(input_ids=ids[:, :190], past_key_values=c)
        for t in range(8):
            m.model(input_ids=ids[:, 190 + t:191 + t], past_key_values=c)

    cache = DynamicCache()
    with decoding()(model):
        decode(model, cache)
    assert checked == [("compress", 194)] * 2 + [("compress", 104)] * 2
    standin = _standin(decoding, decode, monkeypatch)[1]
    assert cache.get_seq_length() == standin.get_seq_length() == 100
    assert _shared(cache, standin) >= 0.97
