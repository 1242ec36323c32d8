"""ExpectedAttention and SnapKV against a float64 evaluation of their formulas, over every kernel instantiation, the
persistent schedules' corner regimes, strided cache layouts and the edges of S / n_sink / window / kernel size.

The fp64 reference takes the same 16-bit inputs and runs on the device (fp64 cuBLAS never uses TF32), one (b, h) row at
a time so that 128k-position rows stay small. Every scored position is checked against it:
  1. <= 1 ulp of the fp64 score rounded once to the cache dtype (SnapKV's ex2.approx.ftz flushes fp32 results below
     2^-126 to zero: there the kernel may also return 0);
  2. no bias per row: |mean((got - ref) / ref)| <= 8 u / sqrt(12 n) over the n >= 500 positions of a row whose reference
     is a normal 16-bit number (u = 2^-7 bf16, 2^-10 fp16). That is 8 standard errors of pure rounding noise; a constant
     factor on a row (a lost softmax partial, a wrong 1/G, a wrong epsilon) misses it by orders of magnitude, although
     it passes the 1-ulp bar and leaves the selection within the row unchanged;
  3. forced positions equal round(max valid score + 1), the reference's sentinel;
  4. compress: the kept set is the lowest-index-ties top-k of the kernel's own scores, K'/V' are exact gathers.
Measured on an H100 80GB HBM3 (132 SMs, 700 W power limit) over every case of this file: at most 1 ulp from the
rounded fp64 score; at most 4e-4 of a case's positions at 1 ulp for ExpectedAttention and 2.1e-3 for SnapKV (fp16,
window 1); the worst row bias is 0.30 of its bound. Each bar is asserted as stated above, not at the measured values.
"""
import re
from pathlib import Path

import pytest
import torch

from oracle import press_oracle as O
from tests.gpu_support import (assert_compress, assert_vs_ref64, ea_inputs, ea_instantiation, ea_ref64, ea_schedule,
                               _forced_head, _forced_tail, _gather, _layout, LAYOUTS, _name, _native, _sm_count,
                               snap_inputs, snap_parts, snap_ref64)

gpu = pytest.mark.gpu
DEV = "cuda:0"
CSRC = Path(__file__).resolve().parent.parent / "kvpress_b200" / "csrc"
DTYPES = [torch.bfloat16, torch.float16]


# ---------------------------------------------------------------------------------------------------
# the launchers' dispatch rules (expected_attention.cu: launch_ea_t, snapkv.cu: launch_snap_d / launch_snap_t)
# ---------------------------------------------------------------------------------------------------
def snap_instantiation(dtype, D: int, G: int, window: int):
    """<T, D, NQP> of snap_stats_kernel / snap_colsum_kernel: the G * window query rows padded to 128 / 256 / 512."""
    nq = G * window
    nqp = 128 if nq <= 128 else (256 if nq <= 256 else 512)
    return (_name(dtype), D, nqp)


# the instantiation sweep: (dtype, D, G) for ExpectedAttention, (dtype, D, G, window) for SnapKV
EA_SWEEP = [(dt, D, G) for dt in DTYPES for D in (64, 128) for G in (1, 2, 3, 4, 8)]
SNAP_SWEEP = [(dt, D, G, w) for dt in DTYPES for D in (64, 128) for G, w in ((1, 64), (2, 64), (3, 50), (4, 64),
                                                                             (7, 64), (8, 64))]


def test_sweep_reaches_every_instantiation():
    """CPU only: the sweeps below run every <T, D, GR> and <T, D, NQP> the sources instantiate, so their coverage
    cannot shrink unnoticed when a grid or a dispatch rule changes."""
    ea_src = (CSRC / "expected_attention.cu").read_text()
    ea_built = {(n, int(d), int(gr)) for d, gr in re.findall(r"launch_ea_logits_t<T, (\d+), (\d+)>\(", ea_src)
                for n in ("bf16", "fp16")}
    sn_src = (CSRC / "snapkv.cu").read_text()
    sn_built = {(n, int(d), int(q)) for d, q in re.findall(r"KVP_SNAP\((\d+), (\d+)\);", sn_src) for n in ("bf16", "fp16")}
    assert len(ea_built) == 12 and len(sn_built) == 12
    assert {ea_instantiation(*c) for c in EA_SWEEP} == ea_built
    assert {snap_instantiation(*c) for c in SNAP_SWEEP} == sn_built
    # a short last unit (G = 3 -> units of 2 + 1) and two units per kv head (G = 8) are in the grid
    assert any(G % ea_instantiation(dt, D, G)[2] for dt, D, G in EA_SWEEP)
    assert any(G // ea_instantiation(dt, D, G)[2] >= 2 for dt, D, G in EA_SWEEP)


# ---------------------------------------------------------------------------------------------------
# fp64 references
# ---------------------------------------------------------------------------------------------------


# ---------------------------------------------------------------------------------------------------
# the bars
# ---------------------------------------------------------------------------------------------------


# ---------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------


def run_ea(k, v, mu, cov, eps, n_sink, use_vnorm, what, bias=True, n_kept=None):
    """score and compress of one problem, both checked against fp64; returns (scores, ref)."""
    nat = _native()
    S = k.shape[2]
    sc = nat.expected_attention_score(k, v, mu, cov, eps, n_sink, use_vnorm)
    ref = ea_ref64(k, v, mu, cov, eps, n_sink, use_vnorm)
    assert_vs_ref64(sc, ref, _forced_head(S, n_sink), what, bias=bias)
    n_kept = max(1, O.kept_count(S, 0.5)) if n_kept is None else n_kept
    k_out, v_out, idx, sc2 = nat.expected_attention_compress(k, v, mu, cov, eps, n_sink, use_vnorm, n_kept,
                                                             return_indices=True, return_scores=True)
    assert torch.equal(sc2, sc), f"{what}: compress scores differ from the score path"
    assert_compress(k, v, k_out, v_out, idx, sc2, n_kept)
    return sc, ref


def run_snap(k, v, q, window, ksz, what, bias=True):
    nat = _native()
    S = k.shape[2]
    sc = nat.snapkv_score(k, q, window, ksz)
    ref = snap_ref64(q, k, window, ksz)
    assert_vs_ref64(sc, ref, _forced_tail(S, window), what, ftz=True, bias=bias)
    n_kept = max(1, O.kept_count(S, 0.5))
    k_out, v_out, idx, sc2 = nat.snapkv_compress(k, v, q, window, ksz, n_kept, return_indices=True, return_scores=True)
    assert torch.equal(sc2, sc), f"{what}: compress scores differ from the score path"
    assert_compress(k, v, k_out, v_out, idx, sc2, n_kept)
    return sc, ref


# ---------------------------------------------------------------------------------------------------
# 1. the fp64 reference itself
# ---------------------------------------------------------------------------------------------------
def _rel_close(a: torch.Tensor, b: torch.Tensor, rel: float) -> bool:
    """a == b at the forced (+inf) positions, |a - b| <= rel |b| elsewhere"""
    a, b = a.cpu().double(), b.cpu().double()
    fin = torch.isfinite(b)
    return bool(torch.equal(a[~fin], b[~fin]) and ((a[fin] - b[fin]).abs() <= rel * b[fin].abs()).all())


@gpu
def test_fp64_reference_device_matches_cpu():
    k, v, mu, cov = (t.cpu() for t in ea_inputs(2, 2, 3, 300, 64, torch.bfloat16, 1))
    for c, vn, eps in ((cov, True, 1e-2), (None, False, 0.0)):
        dev = ea_ref64(k.to(DEV), v.to(DEV), mu.to(DEV), None if c is None else c.to(DEV), eps, 5, vn)
        assert _rel_close(dev, ea_ref64(k, v, mu, c, eps, 5, vn), 1e-12)
    # and it is the oracle's fp32 formula, to fp32 accuracy
    assert _rel_close(O.expected_attention_scores_fp32(k, v, mu, cov, 0.0, 4, True),
                      ea_ref64(k, v, mu, cov, 0.0, 4, True), 1e-5)
    k, v, q = (t.cpu() for t in snap_inputs(2, 2, 3, 300, 64, 16, torch.float16, 2))
    cpu = snap_ref64(q, k, 16, 5)
    assert _rel_close(snap_ref64(q.to(DEV), k.to(DEV), 16, 5), cpu, 1e-12)
    assert _rel_close(O.snapkv_scores_fp32(q, k, 16, 5), cpu, 1e-5)


# ---------------------------------------------------------------------------------------------------
# 2. instantiation sweep
# ---------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype,D,G", EA_SWEEP, ids=[f"{_name(dt)}-d{D}-g{G}" for dt, D, G in EA_SWEEP])
def test_ea_instantiations(dtype, D, G):
    k, v, mu, cov = ea_inputs(2, 2, G, 2500, D, dtype, 100 + 10 * D + G)
    run_ea(k, v, mu, cov, 0.0, 4, True, f"ea {ea_instantiation(dtype, D, G)} G={G}")


EA_VARIANTS = [(dt, D, cov, vn, eps) for dt in DTYPES for D, cov, vn, eps in (
    (128, True, False, 0.0), (64, True, True, 1e-2), (128, True, False, 1e-2),
    (32, False, True, 0.0), (64, False, True, 1e-2), (96, False, False, 0.0), (128, False, True, 0.0),
    (256, False, True, 1e-2))]


@gpu
@pytest.mark.parametrize("dtype,D,cov,use_vnorm,eps", EA_VARIANTS,
                         ids=[f"{_name(a)}-d{b}-{'cov' if c else 'nocov'}-{'vn' if d else 'novn'}-eps{e}"
                              for a, b, c, d, e in EA_VARIANTS])
def test_ea_score_variants(dtype, D, cov, use_vnorm, eps):
    """covariance x use_vnorm x epsilon, and the covariance-free kernel at every rows-per-lane branch (D = 32: LPR 4,
    64: 8, 96 / 128: 16, 256: 32)."""
    k, v, mu, c = ea_inputs(2, 2, 3, 2500, D, dtype, 200 + D, cov=cov)
    run_ea(k, v, mu, c, eps, 4, use_vnorm, f"ea {_name(dtype)} D={D} cov={cov} vnorm={use_vnorm} eps={eps}")


@gpu
@pytest.mark.parametrize("dtype,D,G,window", SNAP_SWEEP,
                         ids=[f"{_name(dt)}-d{D}-g{G}-w{w}" for dt, D, G, w in SNAP_SWEEP])
def test_snapkv_instantiations(dtype, D, G, window):
    k, v, q = snap_inputs(2, 2, G, 2500, D, window, dtype, 300 + D + G)
    run_snap(k, v, q, window, 5, f"snapkv {snap_instantiation(dtype, D, G, window)} G={G} w={window}")


SNAP_EDGES = [(dt, G, w, S, ksz) for dt in DTYPES for G, w, S, ksz in (
    (4, 64, 2000, 1), (4, 64, 2000, 3), (2, 32, 2000, 7), (4, 1, 1500, 5), (1, 1, 700, 3), (4, 64, 65, 5),
    (2, 16, 17, 7), (8, 64, 129, 5))]


@gpu
@pytest.mark.parametrize("dtype,G,window,S,kernel_size", SNAP_EDGES,
                         ids=[f"{_name(a)}-g{b}-w{c}-s{d}-k{e}" for a, b, c, d, e in SNAP_EDGES])
def test_snapkv_kernel_sizes_and_windows(dtype, G, window, S, kernel_size):
    """kernel_size 1 / 3 / 7, window 1, and S = window + 1 (one scored position)."""
    k, v, q = snap_inputs(1, 2, G, S, 128, window, dtype, 400 + S + kernel_size)
    run_snap(k, v, q, window, kernel_size, f"snapkv {_name(dtype)} G={G} w={window} S={S} k={kernel_size}")


SNAP_MHA = [(dt, D, w) for dt in DTYPES for D in (64, 128) for w in (257, 384, 511)]


@gpu
@pytest.mark.parametrize("dtype,D,window", SNAP_MHA, ids=[f"{_name(a)}-d{b}-w{c}" for a, b, c in SNAP_MHA])
def test_snapkv_one_query_head_per_kv_head_windows_above_256(dtype, D, window):
    """Multi-head attention (G = 1) with windows of 257 to 511: the 512-row instantiation with up to half of its rows
    padding, as a process's first call (the per-stream workspaces dropped, so none is larger than this call asks)."""
    _native()._WS_CACHE.clear()
    k, v, q = snap_inputs(3, 1, 1, 1500, D, window, dtype, 800 + window + D)
    run_snap(k, v, q, window, 5, f"snapkv {snap_instantiation(dtype, D, 1, window)} G=1 w={window}")


@gpu
def test_snapkv_press_window_300_on_a_multi_head_llama():
    """SnapKVPress(window_size=300) on a multi-head-attention model, as the first call of the process's workspaces."""
    from transformers import DynamicCache

    from kvpress_b200 import SnapKVPress
    from kvpress_b200.presses.scorer_press import kept_count
    from tests.tiny_models import tiny_llama

    nat = _native()
    model = tiny_llama(dtype=torch.bfloat16, device=DEV, head_dim=128, heads=4, kv_heads=4)
    ids = torch.randint(2, 250, (1, 1000), device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))
    full = DynamicCache()
    model.model(input_ids=ids, past_key_values=full)
    nat._WS_CACHE.clear()
    cache = DynamicCache()
    with SnapKVPress(compression_ratio=0.5, window_size=300)(model):
        model.model(input_ids=ids, past_key_values=cache)
    n_kept = kept_count(1000, 0.5)
    assert cache.get_seq_length() == n_kept
    for lf, lc in zip(full.layers, cache.layers):
        # the window is kept, and every kept row is a row of the full cache (values are gathered as they are)
        assert torch.equal(lc.values[:, :, n_kept - 300:], lf.values[:, :, -300:])
        hit = (lc.values[:, :, :, None, :] == lf.values[:, :, None, :, :]).all(-1).any(-1)
        assert hit.all(), "a kept value row is not a row of the full cache"


# ---------------------------------------------------------------------------------------------------
# 3. persistent schedules: each shape asserts the regime it is meant to reach on this device
# ---------------------------------------------------------------------------------------------------
def _crosses(lo, hi, n_tp):
    """the range [lo, hi) holds items of more than one unit"""
    return lo // n_tp != (hi - 1) // n_tp


EA_REGIMES = {
    # name: (B, H, G, S)
    "one_tile_per_cta": (1, 2, 4, 2500),
    "ranges_cross_units": (4, 8, 4, 1000),
    "unit_over_many_ctas": (1, 5, 4, 12700),
    "g8_rows_over_sm_count": (18, 8, 8, 700),
}


@gpu
@pytest.mark.parametrize("regime", list(EA_REGIMES))
def test_ea_schedule_regimes(regime):
    B, H, G, S = EA_REGIMES[regime]
    n_tp, n_workers, ranges, spans = ea_schedule(B * H, G, S)
    sm = _sm_count()
    if regime == "one_tile_per_cta":
        assert n_workers < sm and all(hi - lo == 1 for lo, hi in ranges)
    elif regime == "ranges_cross_units":
        assert sum(_crosses(lo, hi, n_tp) for lo, hi in ranges) >= 10
    elif regime == "unit_over_many_ctas":
        assert min(c for _, c in spans) >= 3
        assert any(lo % n_tp != 0 and _crosses(lo, hi, n_tp) and hi % n_tp != 0 for lo, hi in ranges)
    else:
        assert B * H > sm and G // ea_instantiation(torch.bfloat16, 128, G)[2] == 2
    k, v, mu, cov = ea_inputs(B, H, G, S, 128, torch.bfloat16, 500 + S)
    run_ea(k, v, mu, cov, 0.0, 4, True, f"ea schedule {regime}")


@gpu
def test_ea_llama8b_128k_every_row_vs_fp64():
    """The Llama-3.1-8B layer at 128k (Hq 32, Hkv 8, D 128): every score of every kv head against fp64."""
    B, H, G, S = 1, 8, 4, 131072
    n_tp, n_workers, ranges, spans = ea_schedule(B * H, G, S)
    assert min(c for _, c in spans) >= 3
    k, v, mu, cov = ea_inputs(B, H, G, S, 128, torch.bfloat16, 41)
    run_ea(k, v, mu, cov, 0.0, 4, True, "ea llama8b 128k", n_kept=O.kept_count(S, 0.7))


SNAP_REGIMES = {
    # name: (B, H, G, window, S)
    "empty_trailing_parts": (1, 1, 4, 64, 25500),
    "rows_up_to_sm_count": (12, 8, 4, 32, 3000),
    "rows_over_sm_count": (18, 8, 2, 64, 1500),
}


@gpu
@pytest.mark.parametrize("regime", list(SNAP_REGIMES))
def test_snapkv_schedule_regimes(regime):
    B, H, G, w, S = SNAP_REGIMES[regime]
    sm = _sm_count()
    cpr, used1, used2 = snap_parts(B * H, S, w, sm)
    if regime == "empty_trailing_parts":
        assert used1 < cpr and used2 < cpr
    elif regime == "rows_up_to_sm_count":
        assert 67 <= B * H <= sm and cpr == 1
    else:
        assert B * H > sm and cpr == 1
    k, v, q = snap_inputs(B, H, G, S, 128, w, torch.bfloat16, 600 + S)
    run_snap(k, v, q, w, 5, f"snapkv schedule {regime}")


# ---------------------------------------------------------------------------------------------------
# 4. strided layouts: consumed in place, bitwise equal to contiguous copies
# ---------------------------------------------------------------------------------------------------


@gpu
@pytest.mark.parametrize("dtype,D", [(torch.bfloat16, 128), (torch.float16, 64)], ids=["bf16-d128", "fp16-d64"])
@pytest.mark.parametrize("kind", LAYOUTS)
def test_strided_layouts(kind, dtype, D):
    nat = _native()
    B, S, G, w = 3, 1500, 2, 32
    H = 1 if kind == "one_head_of_wider_cache" else 4
    k, v = _layout(kind, B, H, S, D, dtype, 700 + D)
    assert nat._rows_ok(k) and nat._rows_ok(v)
    if kind != "v_strided_k_contiguous":
        assert not k.is_contiguous()
    assert not v.is_contiguous()
    kc, vc = k.contiguous(), v.contiguous()
    _, _, mu, cov = ea_inputs(B, H, G, 8, D, dtype, 701)
    q = snap_inputs(B, H, G, 8, D, w, dtype, 702)[2]
    n_kept = O.kept_count(S, 0.6)

    sc = nat.expected_attention_score(k, v, mu, cov, 1e-2, 4, True)
    assert torch.equal(sc, nat.expected_attention_score(kc, vc, mu, cov, 1e-2, 4, True))
    assert_vs_ref64(sc, ea_ref64(kc, vc, mu, cov, 1e-2, 4, True), _forced_head(S, 4), f"ea layout {kind}")
    assert torch.equal(nat.expected_attention_score(k, v, mu, None, 0.0, 4, True),
                       nat.expected_attention_score(kc, vc, mu, None, 0.0, 4, True))
    got = nat.expected_attention_compress(k, v, mu, cov, 1e-2, 4, True, n_kept, return_indices=True, return_scores=True)
    want = nat.expected_attention_compress(kc, vc, mu, cov, 1e-2, 4, True, n_kept, return_indices=True,
                                           return_scores=True)
    assert all(torch.equal(a, b) for a, b in zip(got, want))
    assert_compress(kc, vc, *got, n_kept)

    sc = nat.snapkv_score(k, q, w, 5)
    assert torch.equal(sc, nat.snapkv_score(kc, q, w, 5))
    assert_vs_ref64(sc, snap_ref64(q, kc, w, 5), _forced_tail(S, w), f"snapkv layout {kind}", ftz=True)
    got = nat.snapkv_compress(k, v, q, w, 5, n_kept, return_indices=True, return_scores=True)
    want = nat.snapkv_compress(kc, vc, q, w, 5, n_kept, return_indices=True, return_scores=True)
    assert all(torch.equal(a, b) for a, b in zip(got, want))
    assert_compress(kc, vc, *got, n_kept)


# ---------------------------------------------------------------------------------------------------
# 5. ExpectedAttention edges
# ---------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("n_sink", [0, 1, 127, 128, 129, 999])
def test_ea_n_sink(n_sink):
    k, v, mu, cov = ea_inputs(1, 2, 4, 1000, 128, torch.bfloat16, 800 + n_sink)
    run_ea(k, v, mu, cov, 0.0, n_sink, True, f"ea n_sink={n_sink}")


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("S", [1, 2, 127, 128, 129, 257])
def test_ea_short_caches(S, dtype):
    for cov in (True, False):
        k, v, mu, c = ea_inputs(2, 2, 2, S, 64, dtype, 900 + S, cov=cov)
        run_ea(k, v, mu, c, 0.0, 0, True, f"ea {_name(dtype)} S={S} cov={cov} n_sink=0")
        if S > 4:
            run_ea(k, v, mu, c, 0.0, 4, False, f"ea {_name(dtype)} S={S} cov={cov} n_sink=4")


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_ea_peaked_softmax_across_ctas(dtype):
    """Logits spanning about 60 over one unit spread over many CTAs: every CTA's partial has a different running max."""
    B, H, G, S = 1, 1, 1, 20000
    assert min(c for _, c in ea_schedule(B * H, G, S)[3]) >= 3
    k, v, mu, cov = ea_inputs(B, H, G, S, 128, dtype, 1000, mu_scale=8.5)
    lg = k[0, 0].float() @ mu[0, 0].float() / 128 ** 0.5
    assert 50 < float(lg.max() - lg.min()) < 90
    run_ea(k, v, mu, cov, 0.0, 4, True, f"ea {_name(dtype)} peaked")


@gpu
def test_ea_max_logit_in_last_tile_of_last_cta():
    """The largest logit of every head sits at position S - 1: the last tile of the last CTA of each unit."""
    B, H, G, S, D = 1, 2, 8, 8000, 128
    n_tp, _, ranges, spans = ea_schedule(B * H, G, S)
    assert min(c for _, c in spans) >= 2
    for u, (first, count) in enumerate(spans):
        lo, hi = ranges[first + count - 1]
        assert lo <= (u + 1) * n_tp - 1 < hi  # the unit's last tile belongs to its last CTA
    k, v, mu, cov = ea_inputs(B, H, G, S, D, torch.bfloat16, 1100)
    for h in range(H):
        direction = mu[0, h * G:(h + 1) * G].float().mean(0)
        k[0, h, S - 1] = (direction / direction.norm() * 40.0).to(k.dtype)
    sc, _ = run_ea(k, v, mu, cov, 0.0, 4, True, "ea max logit at S-1")
    assert (sc[0, :, S - 1] == sc[0, :, 4:].max(-1).values).all()


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_ea_identical_keys_tie(dtype):
    """All keys equal: every softmax is uniform, every score ties, compress keeps the sinks and then the lowest
    positions."""
    nat = _native()
    B, H, G, S, n_sink = 2, 2, 4, 3000, 4
    k, v, mu, cov = ea_inputs(B, H, G, S, 128, dtype, 1200)
    k = k[:, :, :1].expand(B, H, S, 128).contiguous()
    sc = nat.expected_attention_score(k, v, mu, cov, 0.0, n_sink, False)
    ref = ea_ref64(k, v, mu, cov, 0.0, n_sink, False)
    assert_vs_ref64(sc, ref, _forced_head(S, n_sink), f"ea {_name(dtype)} identical keys", bias=False)
    assert (sc[..., n_sink:] == sc[0, 0, n_sink]).all()
    for n_kept in (1, 4, 5, 1000, S):
        k_out, v_out, idx, _ = nat.expected_attention_compress(k, v, mu, cov, 0.0, n_sink, False, n_kept,
                                                               return_indices=True)
        assert torch.equal(idx.long(), torch.arange(n_kept, device=DEV).expand(B, H, n_kept))
        assert torch.equal(k_out, _gather(k, idx)) and torch.equal(v_out, _gather(v, idx))


# ---------------------------------------------------------------------------------------------------
# 6. selection in fp16 (its own ordered-key mapping)
# ---------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("kind", ["random", "all_equal", "two_values", "with_inf_nan_zero", "ascending", "subnormal"])
def test_scores_compress_tie_rule_fp16(kind):
    nat = _native()
    torch.manual_seed(6)
    B, H, S, D = 2, 3, 4099, 64
    k = torch.randn(B, H, S, D, dtype=torch.float16)
    v = torch.randn(B, H, S, D, dtype=torch.float16)
    if kind == "random":
        sc = torch.randn(B, H, S)
    elif kind == "all_equal":
        sc = torch.full((B, H, S), 0.5)
    elif kind == "two_values":
        sc = (torch.rand(B, H, S) > 0.5).float()
    elif kind == "ascending":
        sc = torch.arange(S).float().expand(B, H, S).clone()  # above 2048 neighbours round to the same fp16
    elif kind == "subnormal":
        sc = torch.randint(-40, 40, (B, H, S)).float() * 2.0 ** -24
    else:
        sc = torch.randn(B, H, S)
        sc[..., 10] = float("inf")
        sc[..., 11] = float("-inf")
        sc[..., 12] = float("nan")
        sc[..., 13:40] = 0.0
        sc[..., 40:60] = -0.0
        sc[..., 60] = 65504.0
        sc[..., 61] = -65504.0
    sc = sc.to(torch.float16)
    for n_kept in (1, 7, S // 2, S - 1, S):
        k_out, v_out, idx = nat.scores_compress(sc.to(DEV), k.to(DEV), v.to(DEV), n_kept, return_indices=True)
        assert torch.equal(idx.cpu().long(), O.select_lowest_index_ties(sc, n_kept)), (kind, n_kept)
        assert torch.equal(k_out.cpu(), O.gather_rows(k, idx.cpu().long()))
        assert torch.equal(v_out.cpu(), O.gather_rows(v, idx.cpu().long()))
        sel = nat.scores_select(sc.to(DEV), n_kept)
        assert torch.equal(sel, idx)
