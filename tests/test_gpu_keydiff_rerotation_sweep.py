"""KeyDiff scores and the KeyRerotationPress compaction against float64 / exact references, at every kernel
instantiation, merge shape, S edge, planted exact score and cache layout; caller scores through every score stride.

1. KeyDiff (keydiff.cu): `keydiff_anchor_kernel<T, LPR>` writes one partial sum of k / ||k|| per 256-position chunk,
   `keydiff_merge_kernel` sums the partials in a fixed order (G = 1024 / d_pad thread groups, four chains each, then the
   G groups) and takes ||anchor||, `keydiff_score_kernel<T, LPR>` computes -cos(k, anchor) in fp32 and rounds once.
   Cosine similarity does not see the anchor's scale, so a lost partial, a wrong merge chain or a wrong anchor norm
   moves every score of a row by a small relative amount; the bars below are built to see that.

   Reference: `keydiff_ref64`, the formula in float64 on the device from the same 16-bit keys.
   Bar: every score is within 1 ulp of round16(ref), or |got - ref| <= ulp16(got) / 2 + E_s. The second arm is for
   scores near 0, where the fp32 dot product cancels and no ulp bar can hold. E_s is an a-priori bound on the kernel's
   fp32 evaluation error, computed in float64 from the inputs (u = 2^-24, a = the anchor, k^ = k / ||k||):
     * dot and norm chains. Each product carries at most one rounding and each of the <= D additions adds u times the
       partial sum, so |fl(k . a) - k . a| <= (D + c) u sum_d |k_sd a_d|. Divided by ||k_s|| ||a||:
           E_dot = (D + 8) u sum_d |k_sd a_d| / (||k_s|| ||a||);
     * the anchor. a_d is a sum of S terms k^_sd, each with a relative error of about 10 u (the per-key sum of squares,
       sqrt, reciprocal and product). The sum runs through an addition chain of length L, read off the code: LPR fma
       per lane, log2(32 / LPR) xor shuffles, 8 warps in shared memory, ceil(n_chunks / 4G) + 3 adds per merge chain
       (the remainder loop adds up to 3 more), 2 to join the four chains, G groups, and the division by S. So
       |da_d| <= (L + 16) u m_d with m_d = mean_s |k^_sd|. The score moves by
       k . da / (||k|| ||a||) - score * (a . da) / ||a||^2, hence
           E_anchor = (L + 16) u (sum_d |k_sd| m_d / (||k_s|| ||a||) + |ref_s| sum_d |a_d| m_d / ||a||^2);
     * a few relative roundings (sqrt, two divisions, the reciprocal of ||a||, the 8-level tree of ||a||^2):
           E_rel = 24 u |ref_s|.
   E_s = E_dot + E_anchor + E_rel. Each case asserts max E_s <= 2^-8 of the largest |score| of its row (half a bf16
   ulp of the row's scale; it is largest, about 2^-9, for isotropic keys at 66k positions), so the E arm cannot go
   slack unnoticed. Rows with >= 500 normal-range
   positions must also pass the no-row-bias bar of tests/test_gpu_scorer_sweep.py (a wrong anchor norm is a constant
   factor on a row); positions that pass only through the E arm enter it at round16(ref).

   Inputs are randn keys, isotropic (a small anchor: an ill-conditioned problem) or plus a shared offset (||a|| about
   0.5, as with real keys), every key scaled by 2^x with x uniform over many binades, so a kernel that weighted keys
   by their norm fails. Planted cases have exact answers: keys +-2^e e_j (k^ exact, every anchor component an exact
   count / S, every score within 1 ulp of -sign a_j / ||a||, keys on a balanced dim exactly 0), all keys equal (every
   score -1), all keys zero (every score 0, canonical selection). Special rows are checked against the formula in fp32
   on the device (`keydiff_ref32`): an inf or NaN element makes its whole (b, h) row NaN; fp16 keys whose norm passes
   65504 stay finite in fp32; bf16 keys whose fp32 sum of squares overflows get weight 0 in the anchor and score 0.

2. KeyRerotationPress (`copy_rows_k_rerotated<T>` in select_compact.cu): every kept key is rotated by
   delta = j - s positions with the reference's rounding points. The emulation on the device: delta and
   angle = fp32(delta * inv_freq) exactly as the kernel computes them; cos and sin of the angle in float64; every fp32
   value within sincosf's documented 2 ulp (counted in the larger of the two binades an interval may straddle) rounded
   to the cache dtype: one candidate for cos16 and sin16, or two near a 16-bit rounding midpoint; then
   k * cos16 + rotate_half(k) * sin16 with torch ops in the cache dtype, which round each product and the sum as the
   kernel does. Every output element must equal one of the admissible results; V' is an exact gather, `idx` canonical.

3. Caller scores (`keys_from_scores_kernel`, knorm.cu) reach the selection through the (b, h) element strides of the
   score tensor: every other head, a slice along S (2-byte-aligned pointer), broadcast over B or H (stride 0) and a
   transposed tensor (copied) must give results bitwise equal to contiguous copies.

Measured on an H100 80GB HBM3 (400 W power limit) over every case of this file: KeyDiff at most 1 ulp from the rounded
fp64 score on every position the 1-ulp arm decides, at most 0.2 % of a case's positions at 1 ulp; the E arm alone
decides positions in 2 of 142 checks, at most 2.8e-5 of a case, and the largest E_s is 1.4e-3; the worst row bias is
0.27 of its bound. Rerotation: 14751 output elements over the file had two admissible results. Each bar is asserted as
stated above, not at the measured values.
"""
import re
from pathlib import Path

import pytest
import torch

from oracle import press_oracle as O
from tests.conftest import ulp16_diff
from tests.gpu_support import (assert_compress, assert_e_small, assert_keydiff_vs_ref, assert_rerotated, _bits, CHUNK,
                               _gather, kd_chain, kd_chunks, kd_dpad, kd_groups, LANES_PER_ROW, lanes_per_row,
                               keydiff_error_bound,
                               keydiff_ref64, _layout, LAYOUTS, MERGE_THREADS, _name, _native, rope_inv_freq, _same)

gpu = pytest.mark.gpu
DEV = "cuda:0"
CSRC = Path(__file__).resolve().parent.parent / "kvpress_b200" / "csrc"
DTYPES = [torch.bfloat16, torch.float16]


# ---------------------------------------------------------------------------------------------------
# KeyDiff's launch shape (launch_keydiff_t, keydiff_merge_kernel)
# ---------------------------------------------------------------------------------------------------


# ---------------------------------------------------------------------------------------------------
# the cases
# ---------------------------------------------------------------------------------------------------
KD_DIMS = [8, 32, 40, 64, 96, 128, 192, 256]
KD_SWEEP = [(dt, D) for dt in DTYPES for D in KD_DIMS]
KD_S_EDGES = [(dt, D, S) for dt in DTYPES for D in (40, 128) for S in (1, 2, 255, 256, 257)]
# n_chunks around one and four merge groups, and past eight, at G = 32, 8, 4; S leaves the last chunk partial
def chunk_edge_counts(G: int):
    return (G - 1, G, G + 1, 4 * G - 1, 4 * G, 4 * G + 1, 8 * G + 3)


KD_CHUNK_EDGES = [(D, c) for D in (32, 128, 256) for c in chunk_edge_counts(kd_groups(D))]
KD_LARGE = {"128k_bh8": (1, 8, 131072, 128), "bh3072_short_s": (4, 768, 200, 64), "bh2048_s33": (2, 1024, 33, 128)}
# planted exact keys: S with a partial last chunk, a merge remainder loop, and an even count of positions s % 16 == 0
PLANT_S = {32: 40 * CHUNK - 64, 128: 36 * CHUNK - 96, 256: 35 * CHUNK - 32}
PLANT_KINDS = ["all_equal", "all_zero", "inf_rows", "nan_rows", "fp16_norm_overflow", "bf16_sum_of_squares_overflow"]
PLANTED = [(kind, dt) for kind in PLANT_KINDS for dt in DTYPES
           if not (kind.startswith("fp16") and dt != torch.float16) and not (kind.startswith("bf16") and dt != torch.bfloat16)]

RR_DIMS = [16, 32, 48, 64, 80, 96, 112, 128, 256]  # 1 to 8 and 16 16-byte vectors per half row
RR_SWEEP = [(dt, D) for dt in DTYPES for D in RR_DIMS]
INV_FREQ_KINDS = ["theta1e4", "theta5e5", "theta1e6", "yarn_like", "random_first_one"]

SCORE_VIEWS = ["every_other_head", "slice_along_s", "broadcast_over_b", "broadcast_over_h", "transposed"]


def n_kept_values(S: int):
    return sorted({n for n in (1, 257, S // 2, S - 1, S) if 1 <= n <= S})


# ---------------------------------------------------------------------------------------------------
# CPU: the sweeps reach every instantiation the sources build
# ---------------------------------------------------------------------------------------------------
def test_sweeps_reach_every_dispatched_keydiff_and_rerotation_instantiation():
    """The KeyDiff sweep runs every <T, LPR> of the anchor and score kernels, each LPR with and without idle lanes,
    every d_pad of the merge and, at G = 32, 8 and 4, n_chunks on both sides of G and 4G and past 8G; the rerotation
    sweep runs both <T> of the rerotating compaction with 1 to 8 and 16 vectors per half row, odd counts included."""
    kd = (CSRC / "keydiff.cu").read_text()
    lprs = set(LANES_PER_ROW)  # one with_lanes_per_row call launches both passes
    m = re.search(r"d_pad = \(D <= (\d+)\) \? (\d+) : \(D <= (\d+)\) \? (\d+) : \(D <= (\d+)\) \? (\d+) : (\d+);", kd)
    bounds = [int(x) for x in m.groups()]
    pads = {bounds[1], bounds[3], bounds[5], bounds[6]}
    assert pads == {32, 64, 128, 256} and bounds[0::2][:3] == [32, 64, 128]
    assert int(re.search(r"constexpr int kKdMergeThreads = (\d+);", kd).group(1)) == MERGE_THREADS
    assert int(re.search(r"constexpr int kScoreChunk = (\d+);", (CSRC / "knorm_chunk.cuh").read_text()).group(1)) == CHUNK

    built = {(n, lpr) for n in ("bf16", "fp16") for lpr in lprs}
    assert {(_name(dt), lanes_per_row(D)) for dt, D in KD_SWEEP} == built
    for lpr in lprs:  # idle lanes: fewer 8-element pieces per row than lanes
        assert {D // 8 < lpr for _, D in KD_SWEEP if lanes_per_row(D) == lpr} == {True, False}
    assert {kd_dpad(D) for _, D in KD_SWEEP} == pads
    assert all(any(kd_dpad(D) == p and D < p for _, D in KD_SWEEP) for p in pads)
    for G in (32, 8, 4):
        assert {c for D, c in KD_CHUNK_EDGES if kd_groups(D) == G} == set(chunk_edge_counts(G))
    assert all(kd_chunks(S) % (4 * kd_groups(D)) != 0 for D, S in PLANT_S.items())  # the remainder loop runs
    assert all(((S + 15) // 16) % 2 == 0 for S in PLANT_S.values())

    sc = (CSRC / "select_compact.cu").read_text()
    rerot = re.search(r"cudaError_t launch_select_compact_rerotate\(.*?\n}", sc, re.S).group(0)
    assert "with_dtype(dtype" in rerot and "launch_select_compact_t<decltype(t)>(" in rerot  # both <T>
    assert "copy_rows_k_rerotated<TR>(" in sc
    want = {(n, hv) for n in ("bf16", "fp16") for hv in (*range(1, 9), 16)}  # head_dim 16 .. 128, and 256
    assert {(_name(dt), D // 16) for dt, D in RR_SWEEP} == want


# ---------------------------------------------------------------------------------------------------
# KeyDiff references and bars
# ---------------------------------------------------------------------------------------------------


def keydiff_ref32(k: torch.Tensor) -> torch.Tensor:
    """The same formula in fp32, sums of squares included: where they overflow, so does the kernel's."""
    kf = k.float()
    kn = (kf * kf).sum(-1).sqrt()
    a = (kf / kn.clamp_min(1e-12)[..., None]).mean(2, keepdim=True)
    an = (a * a).sum(-1).sqrt().clamp_min(1e-8)
    return -((kf * a).sum(-1) / kn.clamp_min(1e-8) / an)


def _check_workspace(nat, k, v, n_kept, scorer):
    p = nat.make_problem(k, v, n_kept)
    nat.workspace_check(p, scorer, nat._workspace(p, scorer, k.device))


def kd_inputs(B, H, S, D, dtype, kind: str, seed: int):
    """randn keys, isotropic or plus a shared offset of norm sqrt(D / 3) (||anchor|| about 0.5), every key scaled by 2^x,
    x uniform over many binades (fp16: norms within its range and below 1e-3 for some keys)."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    lo, hi = (-20.0, 20.0) if dtype == torch.bfloat16 else (-16.0, 10.0)
    x = torch.randn(B, H, S, D, generator=gen, device=DEV)
    if kind == "offset":
        o = torch.randn(B, H, 1, D, generator=gen, device=DEV)
        x = x + o / o.norm(dim=-1, keepdim=True) * (D / 3) ** 0.5
    scale = torch.exp2(torch.rand(B, H, S, 1, generator=gen, device=DEV) * (hi - lo) + lo)
    k = (x * scale).to(dtype)
    v = torch.randn(B, H, S, D, generator=gen, device=DEV).to(dtype)
    return k, v


def run_keydiff(k, v, what: str, n_list=None, bias: bool = True) -> dict:
    """Score against fp64, then compress at every n_kept: scores bitwise equal to keydiff_score, the canonical
    selection of them, exact gathers, a bitwise-equal second call, and no expired wait."""
    nat = _native()
    S, D = k.shape[2], k.shape[3]
    ref = keydiff_ref64(k)
    E = keydiff_error_bound(k, kd_chain(S, D))
    assert_e_small(E, ref, what)
    sc = nat.keydiff_score(k)
    stats = assert_keydiff_vs_ref(sc, ref, E, what, bias=bias)
    for i, n in enumerate(n_list or n_kept_values(S)):
        out = nat.keydiff_compress(k, v, n, return_indices=True, return_scores=True)
        _check_workspace(nat, k, v, n, nat.SCORER_KEYDIFF)
        assert _same(out[3], sc), f"{what} n_kept={n}: compress scores differ from keydiff_score"
        assert_compress(k, v, *out, n)
        if i == 0:
            again = nat.keydiff_compress(k, v, n, return_indices=True, return_scores=True)
            _check_workspace(nat, k, v, n, nat.SCORER_KEYDIFF)
            assert all(_same(a, b) for a, b in zip(out, again)), f"{what}: two calls differ"
    return stats


# ---------------------------------------------------------------------------------------------------
# 1. KeyDiff
# ---------------------------------------------------------------------------------------------------
@gpu
def test_keydiff_fp64_reference_device_matches_cpu():
    for dt, kind in ((torch.bfloat16, "isotropic"), (torch.float16, "offset")):
        k, _ = kd_inputs(2, 3, 700, 40, dt, kind, 5)
        dev = keydiff_ref64(k)
        cpu = keydiff_ref64(k.cpu())
        assert ((dev.cpu() - cpu).abs() <= 1e-12 * cpu.abs().clamp_min(1e-3)).all()
        # and it is the oracle's fp32 formula, to fp32 accuracy (absolute near 0, where fp32 cancels)
        hi = O.keydiff_scores_fp32(k.cpu()).double()
        assert ((hi - cpu).abs() <= 1e-5 * cpu.abs() + 1e-6).all()
        assert ((keydiff_ref32(k).cpu().double() - cpu).abs() <= 1e-5 * cpu.abs() + 1e-6).all()


@gpu
@pytest.mark.parametrize("dtype,D", KD_SWEEP, ids=[f"{_name(dt)}-d{D}" for dt, D in KD_SWEEP])
def test_keydiff_instantiations(dtype, D):
    B, H, S = 2, 3, 3001
    for kind in ("isotropic", "offset"):
        k, v = kd_inputs(B, H, S, D, dtype, kind, 10 * D + (kind == "offset"))
        run_keydiff(k, v, f"keydiff {_name(dtype)} D={D} LPR={lanes_per_row(D)} d_pad={kd_dpad(D)} {kind}")


@gpu
@pytest.mark.parametrize("dtype,D,S", KD_S_EDGES, ids=[f"{_name(dt)}-d{D}-s{S}" for dt, D, S in KD_S_EDGES])
def test_keydiff_short_rows(dtype, D, S):
    for kind in ("isotropic", "offset"):
        k, v = kd_inputs(2, 3, S, D, dtype, kind, 1000 + S + D)
        run_keydiff(k, v, f"keydiff {_name(dtype)} D={D} S={S} {kind}")


@gpu
@pytest.mark.parametrize("D,n_chunks", KD_CHUNK_EDGES, ids=[f"d{D}-g{kd_groups(D)}-c{c}" for D, c in KD_CHUNK_EDGES])
def test_keydiff_merge_chunk_counts(D, n_chunks):
    S = n_chunks * CHUNK - 37
    dtype = DTYPES[n_chunks % 2]
    assert kd_chunks(S) == n_chunks
    for kind in ("isotropic", "offset"):
        k, v = kd_inputs(1, 2, S, D, dtype, kind, 2000 + n_chunks + D)
        run_keydiff(k, v, f"keydiff {_name(dtype)} D={D} G={kd_groups(D)} n_chunks={n_chunks} {kind}",
                    n_list=[257, S // 2])


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("case", list(KD_LARGE))
def test_keydiff_large(case, dtype):
    B, H, S, D = KD_LARGE[case]
    k, v = kd_inputs(B, H, S, D, dtype, "offset", 3000 + S)
    run_keydiff(k, v, f"keydiff {_name(dtype)} {case}")


def planted_unit_keys(B, H, S, D, dtype, seed):
    """Keys +-2^e e_j: j from the chunk, warp, row-select lanes and iteration that own the position in the anchor
    kernel, on dims 1..D-1; the positions s % 16 == 0 on dim 0 with alternating signs, so that a_0 = 0. Returns
    (k, exact float64 scores, mask of the dim-0 positions)."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    s = torch.arange(S, device=DEV)
    loc = s % CHUNK
    rpw = 32 // lanes_per_row(D)
    p = loc % 32
    j = ((s // CHUNK) * 3 + (loc // 32) * 5 + (p % rpw) * 7 + (p // rpw) * 11) % (D - 1) + 1
    orth = s % 16 == 0
    j = torch.where(orth, 0, j).expand(B, H, S)
    sign = torch.where(torch.rand(B, H, S, generator=gen, device=DEV) < 0.7, 1.0, -1.0)
    sign = torch.where(orth, 1.0 - 2.0 * ((s // 16) % 2), sign)
    # bf16: down to 2^-39, above the anchor's 1e-12 clamp and below the score's 1e-8 clamp
    lo, hi = (-39, 40) if dtype == torch.bfloat16 else (-24, 15)
    e = torch.randint(lo, hi + 1, (B, H, S), generator=gen, device=DEV).double()
    k = torch.zeros(B, H, S, D, dtype=dtype, device=DEV)
    k.scatter_(3, j.unsqueeze(-1), (sign.double() * torch.exp2(e)).to(dtype).unsqueeze(-1))
    cnt = torch.zeros(B, H, D, dtype=torch.float64, device=DEV).scatter_add_(2, j, sign.double())
    a = cnt / S
    clamp = float(torch.tensor(1e-8, dtype=torch.float32))  # the kernel's 1e-8f
    exact = -sign.double() * torch.exp2(e) * a.gather(2, j) / (torch.exp2(e).clamp_min(clamp) * a.norm(dim=-1, keepdim=True))
    return k, exact, orth.expand(B, H, S)


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("D", list(PLANT_S))
def test_keydiff_planted_unit_keys(D, dtype):
    """k^ is exact, every anchor component an exact count / S: every score within 1 ulp of -sign a_j / ||a|| (bf16 keys
    below 1e-8 scaled by the clamp: 2^e / 1e-8), and the keys on the balanced dim 0 (orthogonal to the anchor) exactly 0."""
    nat = _native()
    B, H, S = 2, 3, PLANT_S[D]
    k, exact, orth = planted_unit_keys(B, H, S, D, dtype, 40 + D)
    assert ((keydiff_ref64(k) - exact).abs() <= 1e-7 * exact.abs()).all()  # 1e-8 against the fp32 1e-8f
    v = torch.randn(B, H, S, D, device=DEV).to(dtype)
    sc = nat.keydiff_score(k)
    d = ulp16_diff(sc, exact.to(dtype))
    assert int(d.max()) <= 1, f"D={D}: {int((d > 1).sum())} planted scores beyond 1 ulp (max {int(d.max())})"
    assert (sc[orth] == 0).all(), f"D={D}: keys orthogonal to the anchor do not score 0"
    print(f"[measured] keydiff planted {_name(dtype)} D={D}: max ulp {int(d.max())}, "
          f"1-ulp fraction {float((d == 1).float().mean()):.4f}")
    for n in n_kept_values(S):
        out = nat.keydiff_compress(k, v, n, return_indices=True, return_scores=True)
        _check_workspace(nat, k, v, n, nat.SCORER_KEYDIFF)
        assert _same(out[3], sc)
        assert_compress(k, v, *out, n)


def planted_special(kind, dtype, seed):
    """(k, v) of one special case at D = 128: rows of offset keys with special positions planted in them."""
    B, H, S, D = 2, 3, PLANT_S[128], 128
    k, v = kd_inputs(B, H, S, D, dtype, "offset", seed)
    s = torch.arange(S, device=DEV)
    if kind == "all_equal":
        k = k[:, :, :1].expand(B, H, S, D).contiguous()
    elif kind == "all_zero":
        k = torch.zeros_like(k)
    elif kind in ("inf_rows", "nan_rows"):  # one element of one key in two of the six (b, h) rows
        x = float("inf") if kind == "inf_rows" else float("nan")
        k[0, 1, 5, 3] = x
        k[1, 2, S - 1, D - 1] = -x
    elif kind == "fp16_norm_overflow":  # all elements 6000: the norm 67882 passes 65504; and single 65504s
        k[:, :, s % 23 == 5] = 6000.0
        one = torch.zeros(D, dtype=dtype, device=DEV)
        one[7] = 65504.0
        k[:, :, s % 23 == 11] = one
    else:  # bf16_sum_of_squares_overflow: four elements 2^64 (fp32 sum of squares inf); and single 2^63s
        four = torch.zeros(D, dtype=dtype, device=DEV)
        four[:4] = 2.0 ** 64
        k[:, :, s % 23 == 5] = four
        one = torch.zeros(D, dtype=dtype, device=DEV)
        one[9] = -(2.0 ** 63)
        k[:, :, s % 23 == 11] = one
    return k, v


@gpu
@pytest.mark.parametrize("kind,dtype", PLANTED, ids=[f"{k}-{_name(dt)}" for k, dt in PLANTED])
def test_keydiff_planted_special(kind, dtype):
    """all_equal: every score exactly -1, compress keeps positions 0..n_kept-1. all_zero: every score 0, same selection.
    inf_rows / nan_rows: the reference's fp32 anchor is NaN, so is every score of the row. fp16_norm_overflow: nothing
    overflows in fp32. bf16_sum_of_squares_overflow: those keys weigh 0 in the anchor and score 0. The others are
    checked against the fp32 formula on the device: <= 1 ulp of it, or within ulp16 / 2 + 2 E_s (both carry E_s)."""
    nat = _native()
    k, v = planted_special(kind, dtype, 60 + PLANT_KINDS.index(kind))
    B, H, S, D = k.shape
    sc = nat.keydiff_score(k)
    ref = keydiff_ref32(k).double()
    if kind == "all_equal":
        assert (sc == -1).all()
    elif kind == "all_zero":
        assert (sc == 0).all()
    elif kind in ("inf_rows", "nan_rows"):
        nan_rows = torch.zeros(B, H, dtype=torch.bool, device=DEV)
        nan_rows[0, 1] = nan_rows[1, 2] = True
        assert torch.equal(torch.isnan(ref).any(-1), nan_rows) and torch.isnan(ref[nan_rows]).all()
    elif kind == "fp16_norm_overflow":
        assert torch.isfinite(ref).all() and torch.isinf(k[:, :, 5].norm(dim=-1)).all()
    else:
        over = torch.arange(S, device=DEV) % 23 == 5
        assert torch.isinf(k[:, :, over].float().pow(2).sum(-1)).all() and (ref[:, :, over] == 0).all()
        assert (sc[:, :, over] == 0).all()
    E = keydiff_error_bound(k, kd_chain(S, D))
    assert_keydiff_vs_ref(sc, ref, E, f"keydiff special {kind} {_name(dtype)}", bias=False, e_factor=2.0)
    nan = torch.isnan(sc)
    for n in n_kept_values(S):
        k_out, v_out, idx, sc2 = nat.keydiff_compress(k, v, n, return_indices=True, return_scores=True)
        _check_workspace(nat, k, v, n, nat.SCORER_KEYDIFF)
        assert torch.equal(torch.isnan(sc2), nan) and torch.equal(_bits(sc2)[~nan], _bits(sc)[~nan])
        want = O.select_lowest_index_ties(sc.cpu(), n)
        assert torch.equal(idx.long().cpu(), want), f"{kind} n_kept={n}: not the canonical selection"
        if kind in ("all_equal", "all_zero"):
            assert torch.equal(want, torch.arange(n).expand(B, H, n))
        assert _same(k_out, _gather(k, idx)) and _same(v_out, _gather(v, idx)), f"{kind} n_kept={n}: not exact gathers"


@gpu
@pytest.mark.parametrize("dtype,D", [(torch.bfloat16, 128), (torch.float16, 96)], ids=["bf16-d128", "fp16-d96"])
@pytest.mark.parametrize("kind", LAYOUTS)
def test_keydiff_strided_layouts(kind, dtype, D):
    nat = _native()
    B, S = 3, 1500
    H = 1 if kind == "one_head_of_wider_cache" else 4
    k, v = _layout(kind, B, H, S, D, dtype, 800 + D)
    assert nat._rows_ok(k) and nat._rows_ok(v) and not v.is_contiguous()
    if kind != "v_strided_k_contiguous":
        assert not k.is_contiguous()
    kc, vc = k.contiguous(), v.contiguous()
    sc = nat.keydiff_score(k)
    assert _same(sc, nat.keydiff_score(kc)), f"{kind}: scores differ from contiguous copies"
    E = keydiff_error_bound(kc, kd_chain(S, D))
    assert_keydiff_vs_ref(sc, keydiff_ref64(kc), E, f"keydiff layout {kind} {_name(dtype)}")
    n = O.kept_count(S, 0.4)
    got = nat.keydiff_compress(k, v, n, return_indices=True, return_scores=True)
    want = nat.keydiff_compress(kc, vc, n, return_indices=True, return_scores=True)
    assert all(_same(a, b) for a, b in zip(got, want)), f"{kind}: compress differs from contiguous copies"
    assert_compress(kc, vc, *got, n)


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_keydiff_graph_replay(dtype):
    """A captured compress (memset, anchor, merge, score, select + compact) replayed on new inputs equals an eager call."""
    nat = _native()
    B, H, S, D = 2, 4, 9000, 128
    n = S // 2
    k, v = kd_inputs(B, H, S, D, dtype, "offset", 4000)
    kk, vv = k.clone(), v.clone()
    graphed = nat.capture(lambda: nat.keydiff_compress(kk, vv, n, return_indices=True, return_scores=True))
    k2, v2 = kd_inputs(B, H, S, D, dtype, "isotropic", 4001)
    kk.copy_(k2)
    vv.copy_(v2)
    replayed = [t.clone() for t in graphed.replay()]
    torch.cuda.synchronize()
    eager = nat.keydiff_compress(kk, vv, n, return_indices=True, return_scores=True)
    _check_workspace(nat, kk, vv, n, nat.SCORER_KEYDIFF)
    assert all(_same(a, b) for a, b in zip(replayed, eager)), "graph replay differs from an eager call"
    assert_compress(k2, v2, *replayed, n)
    assert_keydiff_vs_ref(replayed[3], keydiff_ref64(k2), keydiff_error_bound(k2, kd_chain(S, D)),
                          f"keydiff graph replay {_name(dtype)}")


# ---------------------------------------------------------------------------------------------------
# 2. KeyRerotationPress
# ---------------------------------------------------------------------------------------------------


def rr_inputs(B, H, S, D, dtype, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    k = (2 * torch.randn(B, H, S, D, generator=gen, device=DEV)).to(dtype)
    v = torch.randn(B, H, S, D, generator=gen, device=DEV).to(dtype)
    sc = torch.randn(B, H, S, generator=gen, device=DEV).to(dtype)
    return k, v, sc


def _rr(nat, sc, k, v, n, inv):
    out = nat.scores_compress_rerotate(sc, k, v, n, inv, return_indices=True)
    _check_workspace(nat, k, v, n, nat.SCORER_GENERIC)
    return out


@gpu
@pytest.mark.parametrize("dtype,D", RR_SWEEP, ids=[f"{_name(dt)}-d{D}-hv{D // 16}" for dt, D in RR_SWEEP])
def test_rerotation_sweep(dtype, D):
    nat = _native()
    B, H, S = 2, 3, 2000
    k, v, sc = rr_inputs(B, H, S, D, dtype, 5000 + D)
    amb = 0
    for kind in INV_FREQ_KINDS:
        inv = rope_inv_freq(kind, D, D).to(DEV)
        for n in n_kept_values(S):
            out = _rr(nat, sc, k, v, n, inv)
            amb += assert_rerotated(k, v, sc, n, inv, out, f"rerotate {_name(dtype)} D={D} {kind} n_kept={n}")
            if n == S:  # every delta is 0: the identity
                assert _same(out[0], nat.scores_compress(sc, k, v, n)[0]), f"{kind}: n_kept = S is not the identity"
    plain = nat.scores_compress(sc, k, v, S // 2, return_indices=True)
    zero = _rr(nat, sc, k, v, S // 2, torch.zeros(D // 2, device=DEV))
    assert all(_same(a, b) for a, b in zip(zero, plain)), "inv_freq = 0 is not scores_compress"
    print(f"[measured] rerotate {_name(dtype)} D={D}: {amb} elements with two admissible results")


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_rerotation_large_deltas(dtype):
    """n_kept small at S = 128k: |delta| passes 1e5, where sincosf takes its slow argument reduction."""
    nat = _native()
    B, H, S, D = 1, 8, 131072, 128
    k, v, sc = rr_inputs(B, H, S, D, dtype, 5100)
    amb, far = 0, 0
    for kind in ("theta5e5", "random_first_one"):
        inv = rope_inv_freq(kind, D, 7).to(DEV)
        for n in (1, 37, 1000):
            out = _rr(nat, sc, k, v, n, inv)
            far = max(far, int((torch.arange(n, device=DEV) - out[2].long()).abs().max()))
            amb += assert_rerotated(k, v, sc, n, inv, out, f"rerotate 128k {_name(dtype)} {kind} n_kept={n}")
    assert far > 105615  # angles delta * inv_freq[0] = delta past sincosf's fast argument reduction
    print(f"[measured] rerotate 128k {_name(dtype)}: {amb} elements with two admissible results")


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 80])
def test_rerotation_ties_across_tiles(D, dtype):
    """16 tied scores at positions 1272..1287 around the tile boundary 1280, half the others above, half below: with
    n_kept = n_gt + 7, 8, 9 the second tile takes none, none or one tie, and its out_base comes from eq_before."""
    nat = _native()
    B, H, S = 2, 2, 3000
    k, v, _ = rr_inputs(B, H, S, D, dtype, 5200 + D)
    gen = torch.Generator(device=DEV).manual_seed(5201)
    tie = torch.arange(1272, 1288, device=DEV)
    rest = torch.cat([torch.arange(0, 1272, device=DEV), torch.arange(1288, S, device=DEV)])
    order = rest[torch.rand(B, H, rest.numel(), generator=gen, device=DEV).argsort(-1)]
    n_gt = rest.numel() // 2
    sc = torch.zeros(B, H, S, device=DEV)
    sc.scatter_(2, order[..., :n_gt], 1 + torch.rand(B, H, n_gt, generator=gen, device=DEV))
    sc.scatter_(2, order[..., n_gt:], -1 - torch.rand(B, H, rest.numel() - n_gt, generator=gen, device=DEV))
    sc = sc.to(dtype)
    assert (sc[..., tie] == 0).all() and ((sc > 0).sum(-1) == n_gt).all()
    for kind in ("theta1e4", "random_first_one"):
        inv = rope_inv_freq(kind, D, 3).to(DEV)
        for n in (n_gt + 7, n_gt + 8, n_gt + 9):
            out = _rr(nat, sc, k, v, n, inv)
            assert_rerotated(k, v, sc, n, inv, out, f"rerotate ties {_name(dtype)} D={D} {kind} n_kept={n}")


@gpu
@pytest.mark.parametrize("dtype,D", [(torch.bfloat16, 128), (torch.float16, 80)], ids=["bf16-d128", "fp16-d80"])
@pytest.mark.parametrize("kind", LAYOUTS)
def test_rerotation_strided_layouts(kind, dtype, D):
    nat = _native()
    B, S = 3, 1500
    H = 1 if kind == "one_head_of_wider_cache" else 4
    k, v = _layout(kind, B, H, S, D, dtype, 900 + D)
    assert nat._rows_ok(k) and nat._rows_ok(v) and not v.is_contiguous()
    if kind != "v_strided_k_contiguous":
        assert not k.is_contiguous()
    kc, vc = k.contiguous(), v.contiguous()
    sc = torch.randn(B, H, S, device=DEV).to(dtype)
    inv = rope_inv_freq("theta5e5", D).to(DEV)
    n = O.kept_count(S, 0.6)
    got = _rr(nat, sc, k, v, n, inv)
    want = _rr(nat, sc, kc, vc, n, inv)
    assert all(_same(a, b) for a, b in zip(got, want)), f"{kind}: differs from contiguous copies"
    assert_rerotated(kc, vc, sc, n, inv, got, f"rerotate layout {kind} {_name(dtype)}")


# ---------------------------------------------------------------------------------------------------
# 3. caller scores through their (b, h) strides
# ---------------------------------------------------------------------------------------------------
def score_view(kind, B, H, S, dtype, seed):
    """[B, H, S] scores laid out as `kind`, with ties (quarter steps) among them"""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    r = lambda *s: (torch.randn(*s, generator=gen, device=DEV) * 4).round().div(4).to(dtype)  # noqa: E731
    if kind == "every_other_head":
        x = r(B, 2 * H, S)[:, ::2]
        assert x.stride() == (2 * H * S, 2 * S, 1)
    elif kind == "slice_along_s":
        x = r(B, H, S + 1)[..., 1:]
        assert x.data_ptr() % 4 == 2
    elif kind == "broadcast_over_b":
        x = r(1, H, S).expand(B, H, S)
        assert x.stride(0) == 0
    elif kind == "broadcast_over_h":
        x = r(B, 1, S).expand(B, H, S)
        assert x.stride(1) == 0
    else:  # transposed: unit stride along H, copied by the binding
        x = r(B, S, H).transpose(1, 2)
        assert x.stride(2) != 1
    return x


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("kind", SCORE_VIEWS)
def test_caller_score_strides(kind, dtype):
    nat = _native()
    B, H, S, D = 3, 4, 3000, 64
    sc = score_view(kind, B, H, S, dtype, 6000 + SCORE_VIEWS.index(kind))
    scc = sc.contiguous()
    k, v, _ = rr_inputs(B, H, S, D, dtype, 6100)
    inv = rope_inv_freq("theta1e4", D).to(DEV)
    for n in (1, 257, S // 2, S - 1):
        got = nat.scores_compress(sc, k, v, n, return_indices=True)
        _check_workspace(nat, k, v, n, nat.SCORER_GENERIC)
        want = nat.scores_compress(scc, k, v, n, return_indices=True)
        assert all(_same(a, b) for a, b in zip(got, want)), f"{kind} n_kept={n}: scores_compress differs"
        assert_compress(k, v, *got, scc, n)
        sel = nat.scores_select(sc, n)
        assert torch.equal(sel, nat.scores_select(scc, n)) and torch.equal(sel, got[2]), f"{kind} n_kept={n}: scores_select"
        got = _rr(nat, sc, k, v, n, inv)
        want = _rr(nat, scc, k, v, n, inv)
        assert all(_same(a, b) for a, b in zip(got, want)), f"{kind} n_kept={n}: scores_compress_rerotate differs"
        assert_rerotated(k, v, scc, n, inv, got, f"caller scores {kind} {_name(dtype)} n_kept={n}")
