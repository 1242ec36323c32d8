"""CUR on the GPU: the sm_90a kernels (csrc/cur.cu) against a float64 evaluation of their definition
(include/kvpress_b200.h, kvp_cur_score), from the same 16-bit inputs, on the device (tests/cur_backend.py).

With z the float64 score, u = 2^-24 the fp32 unit roundoff and ulp the spacing of the cache dtype: the sinks are exactly
1, NaN sits exactly where z is NaN, and every other score is within 1 ulp of z rounded once, or |score - z| <= ulp / 2 +
E_s, where E_s bounds the kernel's fp32 error before the one rounding. The E_s arm may decide at most 1 % of a case's
positions.

E_s, derived from the kernel's operations (first order; the final factor 1.01 covers the second-order terms). All sums
below are of non-negative terms, so relative errors carry through them as their maximum.
- a = sum_d x_d^2: squares of exact 16-bit inputs in fma chains of 4, two chains added, a butterfly over at most 32
  lanes: at most 10 roundings, rho_a = 10 u.
- with a projection: acc_c = sum_d x_d G_dc, a sequential fma chain, |d acc_c| <= e_c = D u sum_d |x_d G_dc|;
  a = sum_c acc_c^2, another chain: rho_a = (sum_c (2 |acc_c| e_c + e_c^2)) / a + r u.
- window sum W: per lane at most ceil(w / 32) terms in order, then 5 butterfly steps:
  rho_W = max over the window of rho_a + (ceil(w / 32) + 5) u; p = a / W: rho_p = rho_a + rho_W + u. Without local
  approximation p = a.
- u(s): p itself (key, value); (p_k + p_v) / 2: max(rho_pk, rho_pv) + u; p_k p_v: rho_pk + rho_pv + u =: rho_u(s).
- T is summed in fp64 from the fp32 u: rho_T = max_s rho_u(s) (+ 2^-53 terms); the quotient is taken in fp64 and
  rounded to fp32 once: E_s = 1.01 z (rho_u(s) + max_t rho_u(t) + 2 u).
"""
import math
from pathlib import Path

import pytest
import torch
from transformers import DynamicCache

from oracle import press_oracle as O
from tests import cur_backend as CB
from tests.conftest import ulp16_diff
from tests.gpu_support import (assert_compress, gpu_ids, lagkv_inputs, LANES_PER_ROW, lanes_per_row, _masked, _name,
                               _native, _prefill, same16, _shared, tiny_gpu_llama, ulp_at)

gpu = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24
WINDOW_MAX, RANK_MAX = 1024, 32
TYPES = CB.LEVERAGE_TYPES
ROOT = Path(__file__).resolve().parent.parent


def projection(D: int, r: int, seed: int) -> torch.Tensor:
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn((D, r), generator=g, device=DEV) / math.sqrt(r)


# --------------------------------------------------------------------------------------------------
# the bound of the module docstring
# --------------------------------------------------------------------------------------------------
def share_bound(x16, w: int, G):
    """(p64, rho_p) of every position, [B, H, S]."""
    x = x16.double()
    D = x.shape[-1]
    if G is None:
        a = x.square().sum(dim=-1)
        rho = torch.full_like(a, 10 * U)
    else:
        g = G.double()
        acc = x @ g
        e = D * U * (x.abs() @ g.abs())
        a = acc.square().sum(dim=-1)
        rho = (2 * acc.abs() * e + e * e).sum(dim=-1) / a + G.shape[1] * U
    if w == 0:
        return a, rho
    S = a.shape[-1]
    pad = (w - S % w) % w
    aw = torch.nn.functional.pad(a, (0, pad)).unflatten(-1, (-1, w))
    rw = torch.nn.functional.pad(rho.nan_to_num(), (0, pad)).unflatten(-1, (-1, w))
    p = (aw / aw.sum(dim=-1, keepdim=True)).flatten(-2)[..., :S]
    rho_w = (rw.amax(dim=-1, keepdim=True) + (-(-w // 32) + 5) * U).expand_as(rw).flatten(-2)[..., :S]
    return p, rho + rho_w + U


def score_bound(k, v, sinks: int, leverage_type: str, w: int, G):
    """(z, E_s): the float64 scores and the bound on the kernel's fp32 error, [B, H, S]."""
    if leverage_type == "key":
        u, rho = share_bound(k, w, G)
    elif leverage_type == "value":
        u, rho = share_bound(v, w, G)
    else:
        pk, rk = share_bound(k, w, G)
        pv, rv = share_bound(v, w, G)
        u, rho = ((pk + pv) / 2, torch.maximum(rk, rv) + U) if leverage_type == "kv_avg" else (pk * pv, rk + rv + U)
    z = u / u.sum(dim=-1, keepdim=True)
    E = 1.01 * z * (rho + rho.nan_to_num().amax(dim=-1, keepdim=True) + 2 * U)
    z[..., :sinks] = 1.0
    E[..., :sinks] = 0.0
    return z, E


def check(k, v, sinks: int, leverage_type: str, w: int, G, sc, what: str) -> dict:
    """The bars of the module docstring for the scores `sc` of (k, v)."""
    dtype = sc.dtype
    z, E = score_bound(k, v, sinks, leverage_type, w, G)
    assert sc.shape == z.shape and sc.dtype == k.dtype
    assert torch.equal(z.nan_to_num(), CB.cur_scores64(k, v, sinks, leverage_type, w, G).nan_to_num())
    assert (sc[..., :sinks] == 1).all(), f"{what}: sinks"
    nan = torch.isnan(z)
    assert torch.equal(torch.isnan(sc), nan), f"{what}: NaN positions differ"
    g, zz, e = sc[~nan], z[~nan], E[~nan].nan_to_num()
    if g.numel() == 0:
        return {"nan": int(nan.sum())}
    d = ulp16_diff(g, zz.to(dtype))
    near = (g.double() - zz).abs() <= ulp_at(zz, dtype) / 2 + e
    ok = (d <= 1) | near
    assert ok.all(), f"{what}: {int((~ok).sum())} positions beyond both bars (max {int(d.max())} ulp)"
    e_arm = int(((d > 1) & near).sum())
    assert e_arm <= max(1, d.numel() // 100), f"{what}: the E_s arm decides {e_arm} of {d.numel()} positions"
    return {"max_ulp": int(d.max()), "e_arm": e_arm}


def run(k, v, sinks, leverage_type, w, G, what, n_kept=None):
    """score and compress of one problem, checked; returns the scores."""
    nat = _native()
    S = k.shape[2]
    sc = nat.cur_score(k, v, sinks, leverage_type, w, G)
    check(k, v, sinks, leverage_type, w, G, sc, what)
    assert same16(nat.cur_score(k, v, sinks, leverage_type, w, G), sc), f"{what}: two calls differ"
    n_kept = max(1, O.kept_count(S, 0.5)) if n_kept is None else n_kept
    k_out, v_out, idx, sc2 = nat.cur_compress(k, v, sinks, leverage_type, w, G, n_kept, return_indices=True,
                                              return_scores=True)
    assert same16(sc2, sc), f"{what}: compress scores differ from the score call"
    assert_compress(k, v, k_out, v_out, idx, sc2, n_kept)
    return sc


# --------------------------------------------------------------------------------------------------
# every instantiation, every window size, the boundaries of S
# --------------------------------------------------------------------------------------------------
HEAD_DIMS = (8, 16, 40, 64, 72, 96, 128, 200, 256)
SWEEP = [(dt, D) for dt in (torch.bfloat16, torch.float16) for D in HEAD_DIMS]


def test_sweep_reaches_every_lanes_per_row_instantiation():
    """csrc/cur.cu instantiates <dtype, lanes per row> for 4, 8, 16 and 32 lanes, plus one projected kernel per dtype;
    HEAD_DIMS reaches each, with and without idle lanes."""
    src = (ROOT / "kvpress_b200" / "csrc" / "cur.cu").read_text()
    assert set(LANES_PER_ROW) == {lanes_per_row(D) for D in HEAD_DIMS}
    assert {D // 8 == lanes_per_row(D) for D in HEAD_DIMS} == {True, False}
    assert "cur_unit_kernel<T, 4, true>" in src


@gpu
@pytest.mark.parametrize("dtype,D", SWEEP, ids=[f"{_name(dt)}-d{D}" for dt, D in SWEEP])
def test_instantiations(dtype, D):
    k, v = lagkv_inputs(2, 2, 1000 + D, D, dtype, seed=D)
    G = projection(D, 20, D)
    for leverage_type in TYPES:
        for w in (16, 0):
            run(k, v, 4, leverage_type, w, None, f"cur {_name(dtype)} d{D} {leverage_type} w{w}")
        run(k, v, 4, leverage_type, 16, G, f"cur {_name(dtype)} d{D} {leverage_type} projected")


@gpu
@pytest.mark.parametrize("w", [1, 2, 15, 16, 17, 100, 255, 256, 257, 1000, WINDOW_MAX])
def test_window_sizes(w):
    k, v = lagkv_inputs(1, 3, 2 * max(w, 300) + 37, 64, torch.bfloat16, seed=w)
    for leverage_type in ("kv_product", "kv_avg"):
        run(k, v, 4, leverage_type, w, None, f"cur w{w} {leverage_type}")


@gpu
@pytest.mark.parametrize("S", [1, 2, 15, 16, 17, 255, 256, 257, 272, 511, 512, 513, 4099])
def test_sequence_boundaries(S):
    """S through the window (16), unit (256) and tile boundaries, S below the window, and every num_sinks regime."""
    k, v = lagkv_inputs(2, 2, S, 128, torch.float16, seed=S)
    for sinks in (0, 4, S, S + 1):
        for w in (16, 0, 300):
            run(k, v, sinks, "kv_product", w, None, f"cur S{S} sinks{sinks} w{w}")


@gpu
def test_128k_and_many_rows():
    k, v = lagkv_inputs(1, 8, 131072, 128, torch.bfloat16, seed=1)
    run(k, v, 4, "kv_product", 16, None, "cur 128k")
    run(k, v, 4, "kv_product", 16, projection(128, 20, 3), "cur 128k projected")
    del k, v
    k, v = lagkv_inputs(30, 100, 300, 64, torch.bfloat16, seed=2)  # 3000 rows
    sc = run(k, v, 4, "kv_product", 16, None, "cur 3000 rows")
    nat = _native()
    for b, h in ((0, 0), (17, 43), (29, 99)):
        alone = nat.cur_score(k[b:b + 1, h:h + 1], v[b:b + 1, h:h + 1], 4, "kv_product", 16)
        assert same16(alone[0, 0], sc[b, h])


@gpu
def test_a_batch_equals_its_rows_run_alone():
    nat = _native()
    k, v = lagkv_inputs(3, 2, 5000, 128, torch.bfloat16, seed=5)
    G = projection(128, 20, 1)
    for g in (None, G):
        sc = nat.cur_score(k, v, 4, "kv_product", 16, g)
        for b in range(3):
            assert same16(nat.cur_score(k[b:b + 1], v[b:b + 1], 4, "kv_product", 16, g), sc[b:b + 1])


# --------------------------------------------------------------------------------------------------
# projection
# --------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("r", [1, 3, 20, RANK_MAX])
def test_projection_ranks(r):
    for dtype, D in ((torch.bfloat16, 128), (torch.float16, 256), (torch.bfloat16, 40)):
        k, v = lagkv_inputs(1, 2, 1500, D, dtype, seed=r)
        G = projection(D, r, r)
        for leverage_type in TYPES:
            run(k, v, 4, leverage_type, 16, G, f"cur r{r} d{D} {leverage_type}")
        run(k, v, 0, "kv_product", 0, G, f"cur r{r} d{D} global")


@gpu
def test_limits_and_the_press_fallback():
    """A window above 1024 or more than 32 columns is refused by the kernel; the press scores the window with its
    float32 torch evaluation and compresses with the shared selection kernels. The press's draw is torch.randn's."""
    from kvpress_b200 import CURPress

    nat = _native()
    w = WINDOW_MAX + 1
    k, v = lagkv_inputs(1, 2, 2 * w + 11, 64, torch.bfloat16, seed=4)
    with pytest.raises(RuntimeError, match="unsupported shape"):
        nat.cur_score(k, v, 4, "kv_product", w)
    with pytest.raises(RuntimeError, match="unsupported shape"):
        nat.cur_score(k, v, 4, "kv_product", 16, projection(64, RANK_MAX + 1, 0))
    with pytest.raises(RuntimeError, match="bad argument"):
        nat.cur_score(k, v, -1, "kv_product", 16)
    press = CURPress(compression_ratio=0.5, local_window_size=w)
    sc = press.score(None, None, k, v, None, {})
    want = CB.cur_score(k, v, 4, "kv_product", w)
    assert (ulp16_diff(sc, want) <= 1).float().mean() >= 0.99 and (ulp16_diff(sc, want) <= 2).all()
    k_out, v_out = press.compress(None, None, k, v, None, {})
    idx = O.select_lowest_index_ties(sc.cpu(), O.kept_count(k.shape[2], 0.5)).to(DEV)
    assert torch.equal(k_out, O.gather_rows(k, idx)) and torch.equal(v_out, O.gather_rows(v, idx))
    # use_random_leverage: G is randn(D, 20, device) / sqrt(20) of the device's global generator
    press = CURPress(compression_ratio=0.5, use_random_leverage=True)
    torch.manual_seed(77)
    sc = press.score(None, None, k, v, None, {})
    torch.manual_seed(77)
    G = torch.randn(64, 20, device=DEV) / math.sqrt(20)
    assert same16(sc, nat.cur_score(k, v, 4, "kv_product", 16, G))
    check(k, v, 4, "kv_product", 16, G, sc, "cur press draw")


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
    else:  # keys[..., a:b, :], as ChunkPress slices chunks: the windows start at the view's first row
        k, v = k[..., 8:-4, :], v[..., 8:-4, :]
        assert not k.is_contiguous() and nat._rows_ok(k)
    for G in (None, projection(D, 20, 2)):
        sc = run(k, v, 4, "kv_product", 16, G, f"cur {layout}")
        assert same16(sc, nat.cur_score(k.contiguous(), v.contiguous(), 4, "kv_product", 16, G))


@gpu
@pytest.mark.parametrize("regime", ["fewer", "equal", "more"])
def test_schedule_regimes(regime):
    """Units per row fewer than, equal to and more than the CTAs a row gets (csrc/cur.cu, launch_cur_t: 4 per SM over
    the rows): with more, a CTA strides over several units. The same rows inside a larger batch, where each row gets
    fewer CTAs, score bitwise the same."""
    nat = _native()
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    units = {"fewer": 2 * sm, "equal": 4 * sm, "more": 8 * sm + 3}[regime]
    S = units * 256 - 5
    k, v = lagkv_inputs(1, 1, S, 64, torch.float16, seed=units)
    sc = run(k, v, 4, "kv_product", 16, None, f"cur schedule {regime} ({units} units, {sm} SMs)")
    kb, vb = k.expand(1, 7, S, 64).contiguous(), v.expand(1, 7, S, 64).contiguous()  # ceil(4 sm / 7) CTAs per row
    batch = nat.cur_score(kb, vb, 4, "kv_product", 16)
    assert all(same16(batch[:, h:h + 1], sc) for h in range(7))


# --------------------------------------------------------------------------------------------------
# degenerate and special inputs: ordinary inputs with defined outputs
# --------------------------------------------------------------------------------------------------
@gpu
def test_zero_windows_zero_rows_nan_and_inf():
    nat = _native()
    k, v = lagkv_inputs(1, 4, 1000, 64, torch.bfloat16, seed=3)
    k[0, 0, 32:48] = 0                # an all-zero window: 0/0, the whole row NaN but the sinks
    v[0, 1, 5] = 0                    # a zero row inside a non-zero window: scores 0
    v[0, 2, 700, 3] = float("nan")    # a NaN input: its row NaN
    sc = run(k, v, 4, "kv_product", 16, None, "cur degenerate")
    assert torch.isnan(sc[0, 0, 4:]).all() and (sc[0, 0, :4] == 1).all()
    assert sc[0, 1, 5] == 0 and torch.isfinite(sc[0, 1]).all()
    assert torch.isnan(sc[0, 2, 4:]).all() and torch.isfinite(sc[0, 3]).all()
    assert torch.isfinite(run(k, v, 4, "value", 16, None, "cur degenerate value")[0, 0]).all()  # K is not read
    assert torch.isfinite(run(k, v, 4, "kv_product", 0, None, "cur degenerate global")[0, :2]).all()
    # all-zero caches: NaN with or without windows
    zk = torch.zeros_like(k)
    for w in (16, 0):
        sc = nat.cur_score(zk, zk, 4, "kv_avg", w)
        assert torch.isnan(sc[..., 4:]).all() and (sc[..., :4] == 1).all()
    # an inf input: inside a window inf / inf = NaN, so its row is NaN; without windows T is inf, the position itself
    # is inf / inf = NaN and every other position of the row is x / inf = 0
    k, v = lagkv_inputs(1, 2, 600, 64, torch.float16, seed=6)
    k[0, 1, 100, 0] = float("inf")
    sc = run(k, v, 4, "key", 16, None, "cur inf local")
    assert torch.isnan(sc[0, 1, 4:]).all() and torch.isfinite(sc[0, 0]).all()
    sc = nat.cur_score(k, v, 4, "key", 0)
    assert torch.isnan(sc[0, 1, 100]) and (sc[0, 1, 4:100] == 0).all() and (sc[0, 1, 101:] == 0).all()
    assert same16(sc, CB.cur_score(k, v, 4, "key", 0))


@gpu
def test_values_near_the_top_of_the_range():
    """fp16 near 65504: every fp32 intermediate stays finite (65504^2 * 256 squared is 1e24). bf16 scaled to 1e15: the
    squared norms (1e32) are finite, and with windows so is everything after them."""
    k, v = lagkv_inputs(1, 2, 1500, 128, torch.float16, seed=8)
    k = (k.float() / k.float().abs().amax() * 65000).half()
    v = (v.float() / v.float().abs().amax() * 60000).half()
    for w in (16, 0):
        run(k, v, 4, "kv_product", w, None, f"cur fp16 top of range w{w}")
    k, v = lagkv_inputs(1, 2, 1500, 128, torch.bfloat16, seed=9, scale=1e15)
    run(k, v, 4, "kv_product", 16, None, "cur bf16 1e15")


# --------------------------------------------------------------------------------------------------
# compress: ties, edges of n_kept, graph replay, workspace check, memory
# --------------------------------------------------------------------------------------------------
@gpu
def test_planted_exact_ties_go_to_the_lowest_position():
    """Periodic K and V: every window repeats, so every score value occurs once per period; the kept set is the
    stand-in's, with ties to the lowest positions."""
    nat = _native()
    k, v = lagkv_inputs(1, 2, 64, 64, torch.bfloat16, seed=11)
    k, v = k.repeat(1, 1, 20, 1), v.repeat(1, 1, 20, 1)
    sc = run(k, v, 0, "kv_product", 16, None, "cur ties", n_kept=333)
    assert same16(sc[..., :64], sc[..., 64:128]) and sc[0, 0].unique().numel() <= 64
    got = nat.cur_compress(k, v, 0, "kv_product", 16, None, 333, True, True)
    want = CB.cur_compress(k, v, 0, "kv_product", 16, None, 333, True, True)
    if same16(got[3], want[3]):  # identical scores: the selections must be identical
        assert all(torch.equal(a, b) for a, b in zip(got[:3], want[:3]))


@gpu
def test_compress_edges_nullable_outputs_and_n_kept_zero():
    import ctypes

    nat = _native()
    k, v = lagkv_inputs(2, 2, 700, 64, torch.bfloat16, seed=12)
    S = k.shape[2]
    for n_kept in (1, S):
        run(k, v, 4, "kv_product", 16, None, f"cur n_kept {n_kept}", n_kept=n_kept)
    full = nat.cur_compress(k, v, 4, "kv_product", 16, None, 300, True, True)
    bare = nat.cur_compress(k, v, 4, "kv_product", 16, None, 300)
    assert bare[2] is None and bare[3] is None and same16(bare[0], full[0]) and same16(bare[1], full[1])
    p = nat.make_problem(k, v, 0)
    ws = nat._workspace(p, nat.SCORER_CUR, k.device)
    outs = [torch.full((2, 2, 0, 64), 3, dtype=k.dtype, device=DEV) for _ in range(2)]
    idx = torch.full((2, 2, 1), -5, dtype=torch.int32, device=DEV)
    scores = torch.full((2, 2, S), 7, dtype=k.dtype, device=DEV)
    rc = nat.load().kvp_cur_compress(ctypes.byref(p), k.data_ptr(), v.data_ptr(), 4, 3, 16, None, 0,
                                     outs[0].data_ptr(), outs[1].data_ptr(),
                                     ctypes.cast(idx.data_ptr(), ctypes.POINTER(ctypes.c_int32)), scores.data_ptr(),
                                     ws.data_ptr(), ws.numel(), nat._stream())
    torch.cuda.synchronize()
    assert rc == 0 and (idx == -5).all() and (scores == 7).all()
    assert nat.launches_per_compress(p, nat.SCORER_CUR) == 4


@gpu
def test_replays_under_capture_and_workspace_check():
    nat = _native()
    k, v = lagkv_inputs(1, 8, 8000, 128, torch.bfloat16, seed=9)
    G = projection(128, 20, 5)
    call = lambda: (nat.cur_score(k, v, 4, "kv_avg", 16, G),  # noqa: E731
                    *nat.cur_compress(k, v, 4, "kv_product", 16, None, 4000, True, True))
    eager = call()
    g = nat.capture(call)
    out = g.replay()
    torch.cuda.synchronize()
    assert all(same16(a, b) for a, b in zip(out, eager))
    k.copy_(torch.randn_like(k.float()).to(k.dtype))  # inputs updated in place
    v.mul_(-1)
    out = g.replay()
    torch.cuda.synchronize()
    assert all(same16(a, b) for a, b in zip(out, call()))
    assert not torch.equal(out[3], eager[3])
    p = nat.make_problem(k, v, 4000)
    nat.workspace_check(p, nat.SCORER_CUR, nat._workspace(p, nat.SCORER_CUR, k.device))


@gpu
def test_no_intermediate_at_128k():
    """Memory grows by no more than the workspace (which holds u as fp32 [B Hkv, S]) and the outputs: no cache-sized
    temporary."""
    nat = _native()
    B, H, S, D = 1, 8, 131072, 128
    k, v = lagkv_inputs(B, H, S, D, torch.bfloat16, seed=10)
    n_kept = S // 2
    p = nat.make_problem(k, v, n_kept)
    ws = nat.workspace_bytes(p, nat.SCORER_CUR)
    assert ws <= nat.workspace_bytes(p, nat.SCORER_GENERIC) + B * H * S * 4 + (1 << 16)
    nat._WS_CACHE.clear()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    out = nat.cur_compress(k, v, 4, "kv_product", 16, None, n_kept, True, True)
    torch.cuda.synchronize()
    outputs = sum(t.numel() * t.element_size() for t in out if t is not None)
    grown = torch.cuda.max_memory_allocated() - before
    assert grown <= max(ws, 1 << 20) + outputs + (1 << 16), (grown, ws, outputs)


# --------------------------------------------------------------------------------------------------
# presses on a GPU tiny Llama, every native call checked against the float64 definition
# --------------------------------------------------------------------------------------------------
@pytest.fixture
def checked(monkeypatch):
    """Wraps native.cur_score / cur_compress: every call's scores meet the bars, and its selection is canonical."""
    from kvpress_b200 import native

    calls = []
    real_score, real_compress = native.cur_score, native.cur_compress

    def score(keys, values, sinks, leverage_type, w, G=None):
        sc = real_score(keys, values, sinks, leverage_type, w, G)
        check(keys, values, sinks, leverage_type, w, G, sc, "press score call")
        calls.append(("score", keys.shape[2]))
        return sc

    def compress(keys, values, sinks, leverage_type, w, G, n_kept, return_indices=False, return_scores=False):
        k_out, v_out, idx, sc = real_compress(keys, values, sinks, leverage_type, w, G, n_kept, True, True)
        check(keys, values, sinks, leverage_type, w, G, sc, "press compress call")
        assert_compress(keys, values, k_out, v_out, idx, sc, n_kept)
        calls.append(("compress", keys.shape[2]))
        return k_out, v_out, idx if return_indices else None, sc if return_scores else None

    monkeypatch.setattr(native, "cur_score", score)
    monkeypatch.setattr(native, "cur_compress", compress)
    return calls


def _standin(press_factory, forward, monkeypatch):
    """(model, cache) the same press leaves, run through `forward`, with the float64 stand-ins in place of the
    kernels."""
    with monkeypatch.context() as m:
        CB.install(m)
        model, cache = tiny_gpu_llama(), DynamicCache()
        with press_factory()(model):
            forward(model, cache)
    return model, cache


@gpu
@pytest.mark.parametrize("leverage_type", TYPES)
def test_press_on_a_tiny_llama(checked, monkeypatch, leverage_type):
    from kvpress_b200 import CURPress

    ids = gpu_ids()
    factory = lambda: CURPress(compression_ratio=0.5, leverage_type=leverage_type)  # noqa: E731
    model, cache = tiny_gpu_llama(), DynamicCache()
    with factory()(model):
        model.model(input_ids=ids, past_key_values=cache)
    assert cache.get_seq_length() == 120 and checked == [("compress", 240)] * 2
    assert _shared(cache, _standin(factory, _prefill(ids), monkeypatch)[1]) >= 0.97


@gpu
def test_wrapper_presses_on_a_tiny_llama(checked, monkeypatch):
    """AdaKV, KeyRerotation, ChunkPress (chunks of 50: not a multiple of the window), ComposedPress, CriticalKVPress and
    DecodingPress over CURPress: every native call meets the float64 bars (the `checked` fixture), and each press leaves
    what it leaves with the float64 stand-ins, but for the near-ties at its threshold (97 % shared)."""
    from kvpress_b200 import (AdaKVPress, ChunkPress, ComposedPress, CriticalKVPress, CURPress, DecodingPress,
                              KeyRerotationPress, KnormPress)

    ids = gpu_ids()
    model = tiny_gpu_llama()
    cache = DynamicCache()
    ada = lambda: AdaKVPress(CURPress(compression_ratio=0.5))  # noqa: E731
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

    rerotate = lambda: KeyRerotationPress(CURPress(compression_ratio=0.5))  # noqa: E731
    logits = []

    def with_logits(m, c):
        logits.append(m(input_ids=ids, past_key_values=c).logits)

    cache = DynamicCache()
    with rerotate()(model):
        with_logits(model, cache)
    assert cache.get_seq_length() == 120 and torch.isfinite(logits[0].float()).all()
    assert _shared(cache, _standin(rerotate, with_logits, monkeypatch)[1]) >= 0.97

    del checked[:]
    chunk = lambda: ChunkPress(CURPress(compression_ratio=0.5), chunk_length=50)  # noqa: E731
    cache = DynamicCache()
    with chunk()(model):
        _prefill(ids)(model, cache)
    assert cache.get_seq_length() == 120 and checked == ([("score", 50)] * 4 + [("score", 40)]) * 2
    assert _shared(cache, _standin(chunk, _prefill(ids), monkeypatch)[1]) >= 0.97

    for factory, length in (
            (lambda: ComposedPress([CURPress(compression_ratio=0.25), KnormPress(compression_ratio=0.2)]), 144),
            (lambda: CriticalKVPress(CURPress(compression_ratio=0.5)), 120)):
        cache = DynamicCache()
        with factory()(model):
            _prefill(ids)(model, cache)
        assert cache.get_seq_length() == length
        assert _shared(cache, _standin(factory, _prefill(ids), monkeypatch)[1]) >= 0.97

    del checked[:]
    decoding = lambda: DecodingPress(CURPress(), compression_interval=4, target_size=100)  # noqa: E731

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
