"""Parity of the sm_90a path (through the C ABI, kvpress_b200.native -> libkvpress_b200.so) against
the CPU oracle and the golden vectors of the imported reference. Needs an H100: `pytest -m gpu`.

Bars (north_star): Knorm / StreamingLLM — identical retained-index sets (tie-aware where the
reference's own top-k is ambiguous, see oracle.check_selection); attention-based scorers — scores
within 1e-3 relative of the fp32 evaluation of the reference formula (<= 1 ulp of the 16-bit score), and within the
reference's own 16-bit rounding noise of ITS scores: measured <= 2 ulp on every stored golden case (asserted <= 3) and <= 4 ulp
against the oracle evaluated on the box's host, whose bf16 GEMMs vary with the host CPU (asserted <= 8, < 2 % beyond 2 ulp).
"""
import pytest
import torch

from oracle import press_oracle as O
from tests.conftest import ulp16_diff
from tests.gpu_support import _native

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
# Distance of the kernels' scores (fp32 math, ONE rounding) to the reference's own 16-bit scores (rounded at ~7 points).
# Asserted = the measured maximum + 1:
#  * against the STORED goldens (outputs of the imported reference, fixed): measured <= 2 ulp, none beyond 2 -> 3;
#  * against the oracle evaluated on the box's host at test time: the oracle's bf16 CPU GEMMs round differently from host to
#    host (tests/conftest.py), measured 4 ulp with 1.4e-4 of the positions beyond 2 -> the round-1 band of 8 / 2 % is kept.
REF_ULP_BOUND = 3
HOST_ORACLE_ULP_BOUND = 8
# tie band of the kept-set validity check against the reference's STORED scores: a kept position may sit one score distance
# below the kernel's threshold, which itself may sit one score distance below the reference's
SEL_ULP_SLACK = 2 * REF_ULP_BOUND


def _check_compaction(k, v, k_out, v_out, idx):
    """K'/V' must be exactly the rows the returned indices name, ascending, unique."""
    idx = idx.long().cpu()
    assert (idx[..., 1:] > idx[..., :-1]).all(), "indices must be strictly ascending"
    assert torch.equal(k_out.cpu(), O.gather_rows(k.cpu(), idx))
    assert torch.equal(v_out.cpu(), O.gather_rows(v.cpu(), idx))


# ---------------------------------------------------------------------------------------------------
# Knorm
# ---------------------------------------------------------------------------------------------------
def test_knorm_scores_vs_golden(golden):
    nat = _native()
    k = golden.t("keys").to(DEV)
    got = nat.knorm_score(k).cpu()
    ref = golden.t("knorm_scores")
    d = ulp16_diff(got, ref)
    # fp32 summation order may flip a 16-bit rounding on ~1e-5 of elements, never by more than 1 ulp
    assert d.max() <= 1
    assert (d > 0).float().mean() < 1e-3


def test_knorm_compress_vs_golden(golden):
    nat = _native()
    k, v = golden.t("keys").to(DEV), golden.t("values").to(DEV)
    for i, r in enumerate(golden.ratios):
        n_kept = O.kept_count(golden.S, r)
        k_out, v_out, idx, scores = nat.knorm_compress(k, v, n_kept, return_indices=True, return_scores=True)
        assert k_out.shape == (golden.B, golden.Hkv, n_kept, golden.D)
        _check_compaction(k, v, k_out, v_out, idx)
        # the kept set is exactly the canonical (lowest-position ties) selection of the kernel's own scores
        assert torch.equal(idx.cpu().long(), O.select_lowest_index_ties(scores.cpu(), n_kept))
        # and it is a valid top-k of the REFERENCE's scores
        res = O.check_selection(golden.t("knorm_scores"), idx.cpu(), n_kept, ulp_slack=1)
        assert res["ok"], res
        # identical to the reference's own retained set wherever the reference had no ties to break
        ref_sc = golden.t("knorm_scores")
        if torch.equal(scores.cpu(), ref_sc):
            canon = O.select_lowest_index_ties(ref_sc, n_kept)
            assert torch.equal(idx.cpu().long(), canon)


@pytest.mark.parametrize("shape", [(1, 8, 32768, 128), (2, 4, 5000, 128), (3, 2, 1023, 64), (1, 1, 1025, 256),
                                   (1, 2, 777, 96), (2, 2, 64, 32), (1, 3, 1, 128)])
@pytest.mark.parametrize("ratio", [0.1, 0.5, 0.875])
def test_knorm_compress_vs_oracle_random(shape, ratio):
    nat = _native()
    torch.manual_seed(hash((shape, ratio)) % 2**31)
    k = torch.randn(shape, dtype=torch.bfloat16)
    v = torch.randn(shape, dtype=torch.bfloat16)
    n_kept = O.kept_count(shape[2], ratio)
    kd, vd = k.to(DEV), v.to(DEV)
    k_out, v_out, idx, scores = nat.knorm_compress(kd, vd, n_kept, return_indices=True, return_scores=True)
    assert k_out.shape[2] == n_kept
    if n_kept == 0:
        return
    _check_compaction(k, v, k_out, v_out, idx)
    ref_scores = O.knorm_scores(k)
    assert ulp16_diff(scores.cpu(), ref_scores).max() <= 1
    assert torch.equal(idx.cpu().long(), O.select_lowest_index_ties(scores.cpu(), n_kept))
    assert O.check_selection(ref_scores, idx.cpu(), n_kept, ulp_slack=1)["ok"]


@pytest.mark.parametrize("B,H,S,D", [(1, 8, 2560, 128), (1, 8, 4608, 128), (2, 3, 5119, 128), (1, 8, 2560, 64),
                                     (1, 2, 700, 256), (1, 4, 65, 128), (1, 1, 7, 128), (3, 5, 512, 96)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_knorm_decoding_sized_caches(B, H, S, D, dtype):
    """DecodingPress-sized compactions take the one-launch thread-block-cluster kernel (knorm_cluster.cu): the
    configs[3] shapes 2560 -> 2048 and 4608 -> 2048, ragged slices, duplicate keys (forced ties at the threshold),
    n_kept in {1, target, S}, strided views, no scratch involved."""
    nat = _native()
    torch.manual_seed(S * 7 + D)
    wide = torch.randn(B, H, S + 9, D).to(dtype)
    k = wide[:, :, 3:3 + S]                                    # a view: rows keep their stride, heads too
    v = torch.randn(B, H, S, D).to(dtype)
    if S > 40:
        k[:, :, 20:30] = k[:, :, 5:15]                          # exact duplicates -> ties
    kd, vd = wide.to(DEV)[:, :, 3:3 + S], v.to(DEV)
    for n_kept in sorted({1, min(S, 2048), max(1, S - S // 5), S}):
        k_out, v_out, idx, scores = nat.knorm_compress(kd, vd, n_kept, return_indices=True, return_scores=True)
        _check_compaction(k, v, k_out, v_out, idx)
        assert ulp16_diff(scores.cpu(), O.knorm_scores(k.contiguous())).max() <= 1
        assert torch.equal(idx.cpu().long(), O.select_lowest_index_ties(scores.cpu(), n_kept))
        k2, v2, _, _ = nat.knorm_compress(kd, vd, n_kept)       # without the optional outputs
        assert torch.equal(k2, k_out) and torch.equal(v2, v_out)
    p = nat.make_problem(kd, vd, 1)
    assert nat.launches_per_compress(p, 1) == 1                 # one launch, no memset node


def test_knorm_full_size_properties():
    """BASELINE shape [1,8,131072,128]: size-independent properties instead of an element-wise oracle —
    highest-score-kept invariant (reference tests/presses/test_presses.py:143-162), exact gather,
    idempotence of compaction at the same n_kept."""
    nat = _native()
    torch.manual_seed(7)
    S, n_kept = 131072, O.kept_count(131072, 0.5)
    k = torch.randn(1, 8, S, 128, dtype=torch.bfloat16, device=DEV)
    v = torch.randn(1, 8, S, 128, dtype=torch.bfloat16, device=DEV)
    k_out, v_out, idx, scores = nat.knorm_compress(k, v, n_kept, return_indices=True, return_scores=True)
    idxl = idx.long()
    assert (idxl[..., 1:] > idxl[..., :-1]).all()
    assert torch.equal(k_out, k.gather(2, idxl.unsqueeze(-1).expand(-1, -1, -1, 128)))
    assert torch.equal(v_out, v.gather(2, idxl.unsqueeze(-1).expand(-1, -1, -1, 128)))
    # kept scores are the n_kept largest: sorted kept scores == top of the sorted scores
    kept_scores = scores.float().gather(2, idxl).sort(-1).values
    top_scores = scores.float().sort(-1).values[..., -n_kept:]
    assert torch.equal(kept_scores, top_scores)
    # score tensor agrees with torch's own norm on the GPU to 1 ulp
    assert ulp16_diff(scores.cpu(), (-k.norm(dim=-1)).cpu()).max() <= 1
    # compacting the compacted cache with ratio 0 -> same rows (idempotence at n_kept == S')
    k2, v2, idx2, _ = nat.knorm_compress(k_out, v_out, n_kept, return_indices=True)
    assert torch.equal(k2, k_out) and torch.equal(v2, v_out)
    assert torch.equal(idx2.long(), torch.arange(n_kept, device=DEV).expand_as(idx2))


def test_knorm_strided_views_and_fp16():
    """Views as left by pipeline._remove_answer_from_cache (reference pipeline.py:252-265)."""
    nat = _native()
    torch.manual_seed(3)
    big_k = torch.randn(2, 4, 700, 128, dtype=torch.float16, device=DEV)
    big_v = torch.randn(2, 4, 700, 128, dtype=torch.float16, device=DEV)
    k, v = big_k[:, :, :611], big_v[:, 1:3, 5:616]
    k = k[:, 1:3]
    assert not k.is_contiguous()
    n_kept = 300
    k_out, v_out, idx, scores = nat.knorm_compress(k, v, n_kept, return_indices=True, return_scores=True)
    _check_compaction(k, v, k_out, v_out, idx)
    assert ulp16_diff(scores.cpu(), O.knorm_scores(k.cpu())).max() <= 1
    assert k_out.is_contiguous() and v_out.is_contiguous()


# ---------------------------------------------------------------------------------------------------
# StreamingLLM
# ---------------------------------------------------------------------------------------------------
def test_streaming_vs_golden(golden):
    nat = _native()
    k, v = golden.t("keys").to(DEV), golden.t("values").to(DEV)
    for i, r in enumerate(golden.ratios):
        n_kept = O.kept_count(golden.S, r)
        sc = nat.streaming_score(k, n_kept, 4)
        assert torch.equal(sc.cpu(), golden.t(f"streaming_scores_{i}"))
        k_out, v_out, idx = nat.streaming_compress(k, v, n_kept, 4, return_indices=True)
        assert torch.equal(idx.cpu(), golden.t(f"streaming_kept_{i}"))  # identical retained-index sets
        _check_compaction(k, v, k_out, v_out, idx)


@pytest.mark.parametrize("S,ratio,n_sink", [(131072, 0.5, 4), (1000, 0.999, 4), (10, 0.5, 4), (5000, 0.25, 0),
                                            (2049, 0.3, 128)])
def test_streaming_edge_cases(S, ratio, n_sink):
    nat = _native()
    k = torch.randn(1, 2, S, 128, dtype=torch.bfloat16, device=DEV)
    v = torch.randn(1, 2, S, 128, dtype=torch.bfloat16, device=DEV)
    n_kept = O.kept_count(S, ratio)
    k_out, v_out, idx = nat.streaming_compress(k, v, n_kept, n_sink, return_indices=True)
    if n_kept == 0:
        assert k_out.shape[2] == 0
        return
    want = O.streaming_kept(S, n_kept, n_sink).to(torch.int32)
    assert torch.equal(idx.cpu(), want.expand_as(idx))
    # equals top-k of the reference's 0/1 scores with the lowest-position tie rule
    sc = O.streaming_scores(k.cpu(), ratio, n_sink)
    assert torch.equal(O.select_lowest_index_ties(sc, n_kept), want.long().expand(1, 2, -1))
    _check_compaction(k, v, k_out, v_out, idx)


# ---------------------------------------------------------------------------------------------------
# generic scores -> select + compact (what wrapper presses / custom ScorerPress subclasses use)
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["random", "all_equal", "two_values", "with_inf_nan_zero", "ascending"])
def test_scores_compress_tie_rule(kind):
    nat = _native()
    torch.manual_seed(5)
    B, H, S, D = 2, 3, 4099, 64
    k = torch.randn(B, H, S, D, dtype=torch.bfloat16)
    v = torch.randn(B, H, S, D, dtype=torch.bfloat16)
    if kind == "random":
        sc = torch.randn(B, H, S)
    elif kind == "all_equal":
        sc = torch.full((B, H, S), 0.5)
    elif kind == "two_values":
        sc = (torch.rand(B, H, S) > 0.5).float()
    elif kind == "ascending":
        sc = torch.arange(S).float().expand(B, H, S).clone()
    else:
        sc = torch.randn(B, H, S)
        sc[..., 10] = float("inf")
        sc[..., 11] = float("-inf")
        sc[..., 12] = float("nan")
        sc[..., 13:40] = 0.0
        sc[..., 40:60] = -0.0
    sc = sc.to(torch.bfloat16)
    for n_kept in (1, 7, S // 2, S - 1, S):
        k_out, v_out, idx = nat.scores_compress(sc.to(DEV), k.to(DEV), v.to(DEV), n_kept, return_indices=True)
        _check_compaction(k, v, k_out, v_out, idx)
        assert torch.equal(idx.cpu().long(), O.select_lowest_index_ties(sc, n_kept)), (kind, n_kept)


def test_errors_are_loud():
    nat = _native()
    k = torch.randn(1, 2, 128, 64, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        nat.knorm_compress(k, k, 64)
    kf = torch.randn(1, 2, 128, 64, dtype=torch.float32, device=DEV)
    with pytest.raises(RuntimeError, match="bf16/fp16"):
        nat.knorm_compress(kf, kf, 64)
    kd = torch.randn(1, 2, 128, 12, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(RuntimeError, match="unsupported shape"):
        nat.knorm_compress(kd, kd, 64)


# ---------------------------------------------------------------------------------------------------
# attention-based scorers: tolerance helpers
# ---------------------------------------------------------------------------------------------------
def _round_like(x32: torch.Tensor, dtype) -> torch.Tensor:
    return x32.to(dtype)


def _assert_scores_close(got, ref16, hi32, forced: slice, dtype, stored: bool = False):
    """got: kernel scores (16 bit). ref16: the reference's 16-bit scores. hi32: fp32 evaluation of the
    same formula (forced positions = +inf). Bars: <= 1 ulp from the rounded fp32 evaluation (i.e. the
    kernel's fp32 math is within 1e-3 relative of it), and within the reference's own 16-bit rounding
    noise (a handful of ulps) of the reference scores."""
    S = got.shape[-1]
    keep = torch.ones(S, dtype=torch.bool)
    keep[forced] = False
    g, r, h = got[..., keep], ref16[..., keep], hi32[..., keep]
    d_hi = ulp16_diff(g, _round_like(h, dtype))
    assert d_hi.max() <= 1, f"max ulp distance to rounded fp32 evaluation: {int(d_hi.max())}"
    rel = (g.float() - h).abs() / h.abs().clamp_min(1e-30)
    assert rel.max() <= 2.0 ** -8 + 1e-3  # half an ulp of the final rounding + 1e-3 of fp32 math
    d_ref = ulp16_diff(g, r)
    print(f"[measured] vs reference 16-bit scores: max ulp {int(d_ref.max())}, frac > 2 ulp {float((d_ref > 2).float().mean()):.2e}, "
          f"exact {float((d_ref == 0).float().mean()):.3f}")
    bound, tail = (REF_ULP_BOUND, 1e-3) if stored else (HOST_ORACLE_ULP_BOUND, 2e-2)
    assert d_ref.max() <= bound and (d_ref > 2).float().mean() < tail, (int(d_ref.max()), float((d_ref > 2).float().mean()))
    # the forced positions carry the reference's sentinel: round(max + 1)
    sentinel = (g.float().max() + 1).to(dtype)
    assert (got[..., forced] == sentinel).all()


def _jaccard(a: torch.Tensor, b: torch.Tensor, S: int) -> float:
    ma = torch.zeros(a.shape[:-1] + (S,), dtype=torch.bool).scatter_(-1, a.long(), True)
    mb = torch.zeros(b.shape[:-1] + (S,), dtype=torch.bool).scatter_(-1, b.long(), True)
    return float((ma & mb).sum()) / float((ma | mb).sum())


# ---------------------------------------------------------------------------------------------------
# ExpectedAttention
# ---------------------------------------------------------------------------------------------------
def test_expected_attention_scores_vs_golden(golden):
    nat = _native()
    k, v = golden.t("keys").to(DEV), golden.t("values").to(DEV)
    mu, cov = golden.t("ea_mu"), golden.t("ea_cov")
    variants = [
        ("ea_scores", cov, 0.0, True),
        ("ea_scores_nocov_novnorm", None, 0.0, False),
        ("ea_scores_eps", cov, 1e-2, True),
    ]
    for name, c, eps, vn in variants:
        got = nat.expected_attention_score(k, v, mu.to(DEV), None if c is None else c.to(DEV), eps, 4, vn).cpu()
        hi = O.expected_attention_scores_fp32(golden.t("keys"), golden.t("values"), mu, c, eps, 4, vn)
        _assert_scores_close(got, golden.t(name), hi, slice(0, 4), golden.dtype, stored=True)


def test_expected_attention_compress_vs_golden(golden):
    nat = _native()
    k, v = golden.t("keys").to(DEV), golden.t("values").to(DEV)
    mu, cov = golden.t("ea_mu").to(DEV), golden.t("ea_cov").to(DEV)
    ref_scores = golden.t("ea_scores")
    for i, r in enumerate(golden.ratios):
        n_kept = O.kept_count(golden.S, r)
        k_out, v_out, idx, scores = nat.expected_attention_compress(
            k, v, mu, cov, 0.0, 4, True, n_kept, return_indices=True, return_scores=True)
        _check_compaction(k, v, k_out, v_out, idx)
        idx_c = idx.cpu()
        assert torch.equal(idx_c.long(), O.select_lowest_index_ties(scores.cpu(), n_kept))
        assert (idx_c[..., :min(4, n_kept)] == torch.arange(min(4, n_kept))).all()  # sinks are kept
        res = O.check_selection(ref_scores, idx_c, n_kept, ulp_slack=SEL_ULP_SLACK)
        assert res["ok"], res
        assert _jaccard(idx_c, golden.t(f"ea_kept_{i}"), golden.S) > 0.85  # the reference's own 16-bit noise moves a few ranks


def test_expected_attention_llama8b_shape_vs_fp32_oracle():
    """Llama-3.1-8B layer shape (Hq=32, Hkv=8, D=128) at a length the fp32 oracle finishes in seconds."""
    nat = _native()
    torch.manual_seed(21)
    B, H, Hq, S, D = 1, 8, 32, 6000, 128
    k = torch.randn(B, H, S, D, dtype=torch.bfloat16)
    v = torch.randn(B, H, S, D, dtype=torch.bfloat16)
    mu = (0.5 * torch.randn(B, Hq, D)).to(torch.bfloat16)
    a = torch.randn(B, Hq, D, D) / D ** 0.5
    cov = (a @ a.transpose(-1, -2)).to(torch.bfloat16)
    n_kept = O.kept_count(S, 0.7)
    k_out, v_out, idx, scores = nat.expected_attention_compress(
        k.to(DEV), v.to(DEV), mu.to(DEV), cov.to(DEV), 0.0, 4, True, n_kept, return_indices=True, return_scores=True)
    _check_compaction(k, v, k_out, v_out, idx)
    hi = O.expected_attention_scores_fp32(k, v, mu, cov, 0.0, 4, True)
    ref = O.expected_attention_scores(k, v, mu, cov, 0.0, 4, True)
    _assert_scores_close(scores.cpu(), ref, hi, slice(0, 4), torch.bfloat16)
    assert torch.equal(idx.cpu().long(), O.select_lowest_index_ties(scores.cpu(), n_kept))


# ---------------------------------------------------------------------------------------------------
# SnapKV
# ---------------------------------------------------------------------------------------------------
def test_snapkv_scores_vs_golden(golden):
    nat = _native()
    w, ksz = (int(x) for x in golden.z["snap_window"])
    k = golden.t("keys").to(DEV)
    q = golden.t("snap_q_window")
    got = nat.snapkv_score(k, q.to(DEV), w, ksz).cpu()
    hi = O.snapkv_scores_fp32(q, golden.t("keys"), w, ksz)
    _assert_scores_close(got, golden.t("snap_scores"), hi, slice(golden.S - w, golden.S), golden.dtype, stored=True)


def test_snapkv_compress_vs_golden(golden):
    nat = _native()
    w, ksz = (int(x) for x in golden.z["snap_window"])
    k, v = golden.t("keys").to(DEV), golden.t("values").to(DEV)
    q = golden.t("snap_q_window").to(DEV)
    ref_scores = golden.t("snap_scores")
    for i, r in enumerate(golden.ratios):
        n_kept = O.kept_count(golden.S, r)
        k_out, v_out, idx, scores = nat.snapkv_compress(k, v, q, w, ksz, n_kept, return_indices=True,
                                                        return_scores=True)
        _check_compaction(k, v, k_out, v_out, idx)
        idx_c = idx.cpu()
        assert torch.equal(idx_c.long(), O.select_lowest_index_ties(scores.cpu(), n_kept))
        # the observation window is always kept (lowest positions first when n_kept < w)
        if n_kept >= w:
            assert (idx_c[..., -w:] == torch.arange(golden.S - w, golden.S)).all()
        res = O.check_selection(ref_scores, idx_c, n_kept, ulp_slack=SEL_ULP_SLACK)
        assert res["ok"], res
        if n_kept > 2 * w:  # below that the kept set is (mostly) the window, i.e. ties among sentinels
            # random K/Q give nearly flat attention, so the reference's own 16-bit rounding noise
            # reorders many near-equal scores; the tie-aware check above is the real criterion
            assert _jaccard(idx_c, golden.t(f"snap_kept_{i}"), golden.S) > 0.5


@pytest.mark.parametrize("Hq,Hkv,S", [(32, 8, 4500), (64, 8, 3000), (8, 8, 2000)])
def test_snapkv_model_shapes_vs_fp32_oracle(Hq, Hkv, S):
    """Llama-3.1-8B (G=4), Llama-3.1-70B (G=8) and MHA (G=1) head layouts, window 64, kernel 5."""
    nat = _native()
    torch.manual_seed(31 + Hq)
    B, D, w = 1, 128, 64
    k = torch.randn(B, Hkv, S, D, dtype=torch.bfloat16)
    v = torch.randn(B, Hkv, S, D, dtype=torch.bfloat16)
    q = (torch.randn(B, Hq, w, D) * 1.5).to(torch.bfloat16)
    n_kept = O.kept_count(S, 0.5)
    k_out, v_out, idx, scores = nat.snapkv_compress(k.to(DEV), v.to(DEV), q.to(DEV), w, 5, n_kept,
                                                    return_indices=True, return_scores=True)
    _check_compaction(k, v, k_out, v_out, idx)
    hi = O.snapkv_scores_fp32(q, k, w, 5)
    ref = O.snapkv_scores(q, k, w, 5)
    _assert_scores_close(scores.cpu(), ref, hi, slice(S - w, S), torch.bfloat16)
    assert torch.equal(idx.cpu().long(), O.select_lowest_index_ties(scores.cpu(), n_kept))


# ---------------------------------------------------------------------------------------------------
# full BASELINE sizes: size-independent properties (an element-wise CPU oracle would take minutes)
# ---------------------------------------------------------------------------------------------------
def _gather_dev(x, idx):
    return x.gather(2, idx.long().unsqueeze(-1).expand(-1, -1, -1, x.shape[-1]))


def _assert_topk_of_own_scores(scores, idx, n_kept, forced: slice):
    """kept scores == the n_kept largest scores (as multisets), forced positions all kept."""
    s = scores.float().clone()
    s[..., forced] = float("inf")
    kept = s.gather(2, idx.long()).sort(-1).values
    top = s.sort(-1).values[..., -n_kept:]
    assert torch.equal(kept, top)
    idxl = idx.long()
    assert (idxl[..., 1:] > idxl[..., :-1]).all()


def test_expected_attention_128k_properties():
    """BASELINE configs[2]: ExpectedAttentionPress r=0.7, Llama-3.1-8B layer shape, 128k context."""
    nat = _native()
    torch.manual_seed(41)
    B, H, Hq, S, D = 1, 8, 32, 131072, 128
    k = torch.randn(B, H, S, D, dtype=torch.bfloat16, device=DEV)
    v = torch.randn(B, H, S, D, dtype=torch.bfloat16, device=DEV)
    mu = (0.5 * torch.randn(B, Hq, D, device=DEV)).to(torch.bfloat16)
    a = torch.randn(B, Hq, D, D, device=DEV) / D ** 0.5
    cov = (a @ a.transpose(-1, -2)).to(torch.bfloat16)
    n_kept = O.kept_count(S, 0.7)
    assert n_kept == 39321
    k_out, v_out, idx, scores = nat.expected_attention_compress(k, v, mu, cov, 0.0, 4, True, n_kept,
                                                                return_indices=True, return_scores=True)
    assert torch.equal(k_out, _gather_dev(k, idx)) and torch.equal(v_out, _gather_dev(v, idx))
    _assert_topk_of_own_scores(scores, idx, n_kept, slice(0, 4))
    assert (idx[..., :4] == torch.arange(4, device=DEV)).all()
    # spot-check the scores of one kv head on a 4k slice against the fp32 formula evaluated by torch on the GPU
    h, sl = 3, slice(60000, 64096)
    kk = k[0, h].float()
    lg = torch.stack([(kk @ mu[0, 4 * h + g].float()) / D ** 0.5
                      + ((kk @ cov[0, 4 * h + g].float()) * kk).sum(-1) / (2 * D) for g in range(4)])
    lg = lg[:, 4:]
    p = torch.softmax(lg, dim=-1).mean(0) * v[0, h, 4:].float().norm(dim=-1)
    got = scores[0, h, 4:].float()
    rel = ((got - p).abs() / p.clamp_min(1e-30))[sl]
    assert rel.max() < 2 ** -7


def test_snapkv_32k_and_128k_properties():
    """BASELINE configs[1] (32k, Hq=32) and the per-layer shape of configs[4] (128k, Hq=64)."""
    nat = _native()
    for Hq, S in ((32, 32768), (64, 131072)):
        torch.manual_seed(43 + Hq)
        B, H, D, w = 1, 8, 128, 64
        k = torch.randn(B, H, S, D, dtype=torch.bfloat16, device=DEV)
        v = torch.randn(B, H, S, D, dtype=torch.bfloat16, device=DEV)
        q = (torch.randn(B, Hq, w, D, device=DEV) * 1.5).to(torch.bfloat16)
        n_kept = O.kept_count(S, 0.5)
        k_out, v_out, idx, scores = nat.snapkv_compress(k, v, q, w, 5, n_kept, return_indices=True,
                                                        return_scores=True)
        assert torch.equal(k_out, _gather_dev(k, idx)) and torch.equal(v_out, _gather_dev(v, idx))
        _assert_topk_of_own_scores(scores, idx, n_kept, slice(S - w, S))
        assert (idx[..., -w:] == torch.arange(S - w, S, device=DEV)).all()
        # pre-pool column sums of one kv head against torch (fp32) on the GPU, then the 5-tap box filter
        h, G = 5, Hq // H
        qq = q[0, h * G:(h + 1) * G].reshape(G * w, D).float()
        logits = (qq @ k[0, h].float().T) / D ** 0.5
        i = torch.arange(G * w, device=DEV) % w
        mask = torch.arange(S, device=DEV)[None, :] > (S - w + i)[:, None]
        p = torch.softmax(logits.masked_fill(mask, float("-inf")), dim=-1)[:, : S - w]
        col = p.reshape(G, w, -1).mean(1)
        pooled = torch.nn.functional.avg_pool1d(col[None], 5, stride=1, padding=2)[0].mean(0)
        got = scores[0, h, : S - w].float()
        rel = (got - pooled).abs() / pooled.clamp_min(1e-30)
        assert rel.max() < 2 ** -7


def test_expected_attention_eight_heads_per_kv_head():
    """Llama-3.1-70B grouping (Hq/Hkv = 8): two four-head launches of the tensor-core kernel."""
    nat = _native()
    torch.manual_seed(47)
    B, H, Hq, S, D = 1, 2, 16, 3000, 128
    k = torch.randn(B, H, S, D, dtype=torch.bfloat16)
    v = torch.randn(B, H, S, D, dtype=torch.bfloat16)
    mu = (0.5 * torch.randn(B, Hq, D)).to(torch.bfloat16)
    a = torch.randn(B, Hq, D, D) / D ** 0.5
    cov = (a @ a.transpose(-1, -2)).to(torch.bfloat16)
    got = nat.expected_attention_score(k.to(DEV), v.to(DEV), mu.to(DEV), cov.to(DEV), 0.0, 4, True).cpu()
    hi = O.expected_attention_scores_fp32(k, v, mu, cov, 0.0, 4, True)
    ref = O.expected_attention_scores(k, v, mu, cov, 0.0, 4, True)
    _assert_scores_close(got, ref, hi, slice(0, 4), torch.bfloat16)


# ---------------------------------------------------------------------------------------------------
# KeyRerotationPress (SURVEY §8f row 1): selection + compaction with the K rows re-rotated
# ---------------------------------------------------------------------------------------------------
def _assert_rerotated_close(got: torch.Tensor, ref: torch.Tensor, src_rows: torch.Tensor):
    """cos/sin come from CUDA's sincosf here and from the host libm in the reference run: an fp32 last-bit
    difference can flip the 16-bit rounding of cos or sin, which moves a product by one 16-bit ulp. So:
    nearly all elements bit-exact, the rest within 2^-6 of the row's largest |k| (2 ulp at that scale)."""
    got, ref = got.cpu(), ref.cpu()
    exact = (got.view(torch.int16) == ref.view(torch.int16)).float().mean().item()
    assert exact > 0.995, exact
    bound = src_rows.cpu().float().abs().amax(-1, keepdim=True) * 2.0 ** -6
    assert ((got.float() - ref.float()).abs() <= bound).all()


def test_key_rerotation_vs_golden():
    import numpy as np

    from tests.golden.make_golden import digest16
    from tests.support import rerotation_cases
    nat = _native()
    # the reference's re-rotated keys are stored as digests; the oracle's are bit-identical to them (checked here)
    for tag, S, ratios, (keys_c, values_c, inv_freq_c, scores_c), get in rerotation_cases():
        keys, values, scores, inv_freq = keys_c.to(DEV), values_c.to(DEV), scores_c.to(DEV), inv_freq_c.to(DEV)
        for i, r in enumerate(ratios):
            n_kept = O.kept_count(S, r)
            k2, v2, idx = nat.scores_compress_rerotate(scores, keys, values, n_kept, inv_freq, return_indices=True)
            ref_idx = O.select_lowest_index_ties(scores_c, n_kept)
            assert torch.equal(idx.long().cpu(), ref_idx)
            assert torch.equal(v2.cpu(), O.gather_rows(values_c, ref_idx))
            ref_k = O.rerotate_keys(keys_c, ref_idx, inv_freq_c)
            assert np.array_equal(digest16(ref_k), get(f"perm_k_{i}"))
            _assert_rerotated_close(k2, ref_k, O.gather_rows(keys_c, ref_idx))
            # the Knorm-wrapped golden: same kept set whenever the reference's top-k had no threshold tie
            kn_idx = torch.from_numpy(get(f"knorm_idx_{i}").copy()).long()
            kn_scores = nat.knorm_score(keys)
            k3, _, idx3 = nat.scores_compress_rerotate(kn_scores, keys, values, n_kept, inv_freq, return_indices=True)
            O.check_selection(kn_scores.cpu(), idx3.long().cpu(), n_kept)
            if torch.equal(idx3.long().cpu(), kn_idx):
                ref_k3 = O.rerotate_keys(keys_c, kn_idx, inv_freq_c)
                assert np.array_equal(digest16(ref_k3), get(f"knorm_k_{i}"))
                _assert_rerotated_close(k3, ref_k3, O.gather_rows(keys_c, kn_idx))


@pytest.mark.parametrize("shape,theta", [((1, 4, 8192, 128), 500000.0), ((2, 2, 3001, 64), 10000.0),
                                         ((1, 8, 40000, 128), 10000.0), ((1, 2, 777, 256), 1e6)])
@pytest.mark.parametrize("ratio", [0.3, 0.9])
def test_key_rerotation_vs_oracle_random(shape, theta, ratio):
    nat = _native()
    B, H, S, D = shape
    g = torch.Generator().manual_seed(S + D)
    keys, values = (torch.randn(shape, generator=g).to(torch.bfloat16).to(DEV) for _ in range(2))
    scores = torch.randn(B, H, S, generator=g).to(torch.bfloat16).to(DEV)
    inv_freq = 1.0 / (theta ** (torch.arange(0, D, 2).float() / D))
    n_kept = O.kept_count(S, ratio)
    k2, v2, idx = nat.scores_compress_rerotate(scores, keys, values, n_kept, inv_freq.to(DEV), return_indices=True)
    ref_idx = O.select_lowest_index_ties(scores.cpu(), n_kept)
    assert torch.equal(idx.long().cpu(), ref_idx)
    ref_k, ref_v, _ = O.rerotate_keys(keys.cpu(), ref_idx, inv_freq), O.gather_rows(values.cpu(), ref_idx), None
    assert torch.equal(v2.cpu(), ref_v)
    _assert_rerotated_close(k2, ref_k, O.gather_rows(keys.cpu(), ref_idx))


def test_key_rerotation_full_size_properties():
    """Llama-8B 128k layer. (1) inv_freq = 0 is the identity rotation: bit-identical to kvp_scores_compress.
    (2) a rotation preserves the norm of every (d, d + D/2) pair up to the 16-bit roundings. (3) rotating the
    compacted keys back by the opposite angle recovers the gathered rows (same tolerance)."""
    nat = _native()
    B, H, S, D = 1, 8, 131072, 128
    g = torch.Generator(device=DEV).manual_seed(3)
    keys = torch.randn(B, H, S, D, generator=g, device=DEV, dtype=torch.float32).to(torch.bfloat16)
    values = torch.randn(B, H, S, D, generator=g, device=DEV, dtype=torch.float32).to(torch.bfloat16)
    scores = torch.randn(B, H, S, generator=g, device=DEV, dtype=torch.float32).to(torch.bfloat16)
    n_kept = O.kept_count(S, 0.7)
    k0, v0, i0 = nat.scores_compress(scores, keys, values, n_kept, return_indices=True)
    k1, v1, i1 = nat.scores_compress_rerotate(scores, keys, values, n_kept, torch.zeros(D // 2, device=DEV),
                                              return_indices=True)
    assert torch.equal(i0, i1) and torch.equal(v0, v1) and torch.equal(k0, k1)
    inv_freq = (1.0 / (500000.0 ** (torch.arange(0, D, 2).float() / D))).to(DEV)
    k2, v2, i2 = nat.scores_compress_rerotate(scores, keys, values, n_kept, inv_freq, return_indices=True)
    assert torch.equal(i0, i2) and torch.equal(v0, v2)
    pair = lambda x: torch.hypot(x[..., : D // 2].float(), x[..., D // 2:].float())  # noqa: E731
    assert torch.allclose(pair(k2), pair(k0), rtol=0, atol=2.0 ** -6 * 6)
    delta = (torch.arange(n_kept, device=DEV)[None, None, :] - i0.long()).float()       # new - old position
    ang = delta[..., None] * inv_freq
    c, s = torch.cos(ang), torch.sin(ang)
    lo, hi = k2[..., : D // 2].float(), k2[..., D // 2:].float()
    back = torch.cat((lo * c + hi * s, hi * c - lo * s), dim=-1)                          # rotate by -angle
    assert (back - k0.float()).abs().max().item() < 0.08
    assert (back - k0.float()).abs().mean().item() < 0.006


@pytest.mark.parametrize("dtype,atol", [(torch.float16, 8e-3), (torch.bfloat16, 6e-2)])
@pytest.mark.parametrize("variant", ["default", "scaled"])
def test_key_rerotation_equals_prune_then_rope(dtype, atol, variant):
    """Semantic check in the spirit of the reference's tests/presses/test_key_rerotation_press_rope.py:20-100:
    RoPE(all keys) -> prune + re-rotate   must equal   prune(pre-RoPE keys) -> RoPE at positions 0..n_kept-1
    up to the 16-bit roundings of the two paths ("scaled": a YaRN-like inv_freq and cos/sin scale)."""
    nat = _native()
    B, H, S, D = 2, 2, 4096, 64
    g = torch.Generator().manual_seed(17)
    pre = (0.5 * torch.randn(B, H, S, D, generator=g)).to(dtype).to(DEV)
    inv_freq = 1.0 / (10000.0 ** (torch.arange(0, D, 2).float() / D))
    scale = 1.0
    if variant == "scaled":
        inv_freq = inv_freq / torch.linspace(1.0, 4.0, D // 2)
        scale = 1.1386
    inv_freq = inv_freq.to(DEV)

    def rope(x, n):
        ang = torch.arange(n, device=DEV).float()[:, None] * inv_freq[None, :]
        emb = torch.cat((ang, ang), dim=-1)
        cos, sin = (emb.cos() * scale).to(dtype), (emb.sin() * scale).to(dtype)
        return x * cos + O.rotate_half(x) * sin

    keys = rope(pre, S)
    values = torch.randn(B, H, S, D, generator=g).to(dtype).to(DEV)
    scores = torch.rand(B, H, S, generator=g).to(dtype).to(DEV)
    n_kept = S // 2
    k2, v2, idx = nat.scores_compress_rerotate(scores, keys, values, n_kept, inv_freq, return_indices=True)
    expect = rope(_gather_dev(pre, idx.long()), n_kept)
    assert torch.allclose(k2.float(), expect.float(), atol=atol, rtol=0)
    assert torch.equal(v2, _gather_dev(values, idx.long()))


@pytest.mark.parametrize("B,H,G,S", [(1, 8, 4, 40000), (4, 2, 4, 40000), (2, 4, 1, 50000), (3, 2, 2, 60000)])
def test_expected_attention_compress_matches_its_score_path_large(B, H, G, S):
    """Multi-batch / multi-head problems well above one wave of tiles: compress with and without scores_out must
    keep the same rows, the outputs must be exact gathers, and the kept set must be the top-k of the scores."""
    nat = _native()
    D, Hq = 128, H * G
    g = torch.Generator(device=DEV).manual_seed(B * 1000 + S)
    mk = lambda *s: torch.randn(*s, generator=g, device=DEV, dtype=torch.float32)  # noqa: E731
    K, V = mk(B, H, S, D).to(torch.bfloat16), mk(B, H, S, D).to(torch.bfloat16)
    mu = (0.5 * mk(B, Hq, D)).to(torch.bfloat16)
    a = mk(B, Hq, D, D) / D ** 0.5
    cov = (a @ a.transpose(-1, -2)).to(torch.bfloat16)
    n_kept = O.kept_count(S, 0.7)
    k1, v1, i1, _ = nat.expected_attention_compress(K, V, mu, cov, 0.0, 4, True, n_kept, return_indices=True)
    k2, v2, i2, sc = nat.expected_attention_compress(K, V, mu, cov, 0.0, 4, True, n_kept, return_indices=True,
                                                     return_scores=True)
    assert torch.equal(k1, _gather_dev(K, i1)) and torch.equal(v1, _gather_dev(V, i1))
    assert (i1[..., 1:] > i1[..., :-1]).all()
    _assert_topk_of_own_scores(sc, i2, n_kept, slice(0, 4))
    same = torch.zeros(B, H, S, dtype=torch.bool, device=DEV)
    same.scatter_(2, i1.long(), True)
    overlap = same.gather(2, i2.long()).float().mean().item()
    assert overlap > 0.999, overlap


# ---------------------------------------------------------------------------------------------------
# selection only (kvp_scores_select) and AdaKV's two-stage head-wise selection
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,n_kept", [((2, 4, 3000), 700), ((1, 1, 8 * 40000), 123457), ((3, 2, 257), 257),
                                          ((1, 8, 131072), 1), ((2, 1, 1000), 0)])
@pytest.mark.parametrize("kind", ["random", "ties"])
def test_scores_select_vs_oracle(shape, n_kept, kind):
    nat = _native()
    g = torch.Generator().manual_seed(shape[2] + n_kept)
    scores = torch.randn(shape, generator=g)
    if kind == "ties":
        scores = (scores * 2).round() / 2
    scores = scores.to(torch.bfloat16)
    idx = nat.scores_select(scores.to(DEV), n_kept)
    assert idx.dtype == torch.int32 and tuple(idx.shape) == (*shape[:2], n_kept)
    assert torch.equal(idx.long().cpu(), O.select_lowest_index_ties(scores, n_kept))


def test_adakv_selection_at_128k():
    """AdaKVPress.compress on a [1, 8, 131072] score tensor: budgets, safeguard, and every pruned score is <= every
    unprotected kept score (tie-aware), checked against a straightforward torch evaluation on the device."""
    from types import SimpleNamespace

    from kvpress_b200 import AdaKVPress, ScorerPress

    B, H, S, ratio, alpha = 1, 8, 131072, 0.7, 0.2
    g = torch.Generator(device=DEV).manual_seed(5)
    # heads with very different score scales so that the cross-head selection is far from uniform
    scores = (torch.randn(B, H, S, generator=g, device=DEV) * torch.logspace(-1, 1, H, device=DEV)[None, :, None])
    scores = scores.to(torch.bfloat16)

    class Fixed(ScorerPress):
        def score(self, *a):
            return scores.clone()

    module = SimpleNamespace(config=SimpleNamespace(_attn_implementation="sdpa"))
    K = torch.empty(B, H, S, 8, device=DEV, dtype=torch.bfloat16)
    press = AdaKVPress(Fixed(compression_ratio=ratio), alpha_safeguard=alpha)
    k2, v2 = press.compress(module, None, K, K, None, {})
    assert k2 is K and v2 is K
    b, h, s = module.masked_key_indices
    n_kept = O.kept_count(S, ratio)
    n_safe = int(n_kept * alpha)
    assert b.numel() == H * (S - n_kept)
    pruned = torch.zeros(B, H, S, dtype=torch.bool, device=DEV)
    pruned[b, h, s] = True
    assert pruned.sum().item() == H * (S - n_kept)                       # triples are distinct
    kept_per_head = (~pruned).sum(-1)
    assert (kept_per_head >= n_safe).all() and kept_per_head.float().std().item() > 100
    # safeguard: the n_safe best positions of every head (canonical tie rule) survive
    safe = O.select_lowest_index_ties(scores.cpu(), n_safe).to(DEV)
    assert not pruned.gather(-1, safe).any()
    # every pruned score <= every kept, unprotected score
    boosted = scores.float().scatter(-1, safe, float("inf"))
    assert boosted[pruned].max().item() <= boosted[~pruned].min().item()


# ---------------------------------------------------------------------------------------------------
# KeyDiffPress (SURVEY §8f row 3)
# ---------------------------------------------------------------------------------------------------
def _assert_keydiff_scores(got: torch.Tensor, keys_cpu: torch.Tensor, ref16=None):
    """Kernel score == fp32 evaluation of the reference formula rounded once (<= 1 ulp; absolute 2^-9 around the
    sign change where ulps shrink to nothing); within REF_ULP_BOUND ulp of the reference's own 16-bit scores."""
    got = got.cpu()
    hi = O.keydiff_scores_fp32(keys_cpu)
    want = hi.to(got.dtype)
    small = hi.abs() < 2.0 ** -5
    assert ulp16_diff(got, want)[~small].max().item() <= 1
    assert (got.float() - hi)[small].abs().max().item() <= 2.0 ** -9 if small.any() else True
    if ref16 is not None:
        d = ulp16_diff(got, ref16)[~small]
        assert d.max().item() <= 8 and (d <= 2).float().mean().item() > 0.97


def test_keydiff_vs_golden():
    import numpy as np

    from tests.conftest import GOLDEN_DIR
    nat = _native()
    z = np.load(GOLDEN_DIR / "keydiff.npz")
    for tag, (B, H, S, D, is_half) in zip("abc", z["cases"]):
        dtype = torch.float16 if is_half else torch.bfloat16
        keys = torch.from_numpy(z[f"{tag}_keys"].copy()).view(dtype)
        ref = torch.from_numpy(z[f"{tag}_scores"].copy()).view(dtype)
        sc = nat.keydiff_score(keys.to(DEV))
        _assert_keydiff_scores(sc, keys, ref)
        values = torch.randn(keys.shape).to(dtype)
        for ratio in (0.25, 0.6):
            n_kept = O.kept_count(int(S), ratio)
            k2, v2, idx, sc2 = nat.keydiff_compress(keys.to(DEV), values.to(DEV), n_kept, return_indices=True,
                                                    return_scores=True)
            assert torch.equal(sc2, sc)
            assert torch.equal(idx.long().cpu(), O.select_lowest_index_ties(sc.cpu(), n_kept))
            _check_compaction(keys, values, k2, v2, idx)
            assert O.check_selection(ref, idx.long().cpu(), n_kept, ulp_slack=8)["ok"]  # KeyDiff: <= 8 ulp asserted above


@pytest.mark.parametrize("shape", [(1, 8, 32768, 128), (2, 3, 5000, 64), (1, 2, 1023, 256), (3, 1, 257, 32)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_keydiff_vs_fp32_oracle_random(shape, dtype):
    nat = _native()
    B, H, S, D = shape
    g = torch.Generator().manual_seed(S + D)
    keys = (torch.randn(shape, generator=g) + 0.7 * torch.randn(B, H, 1, D, generator=g)).to(dtype)
    values = torch.randn(shape, generator=g).to(dtype)
    # a strided view (every other head of a wider cache) must be consumed in place
    wide = torch.zeros(B, 2 * H, S, D, dtype=dtype, device=DEV)
    wide[:, ::2] = keys.to(DEV)
    sc = nat.keydiff_score(wide[:, ::2])
    _assert_keydiff_scores(sc, keys)
    n_kept = O.kept_count(S, 0.5)
    k2, v2, idx, _ = nat.keydiff_compress(wide[:, ::2], values.to(DEV), n_kept, return_indices=True)
    assert torch.equal(idx.long().cpu(), O.select_lowest_index_ties(sc.cpu(), n_kept))
    _check_compaction(keys, values, k2, v2, idx)


def test_keydiff_128k_properties():
    nat = _native()
    B, H, S, D = 1, 8, 131072, 128
    g = torch.Generator(device=DEV).manual_seed(9)
    k = (torch.randn(B, H, S, D, generator=g, device=DEV) + torch.randn(B, H, 1, D, generator=g, device=DEV)).to(torch.bfloat16)
    v = torch.randn(B, H, S, D, generator=g, device=DEV).to(torch.bfloat16)
    n_kept = O.kept_count(S, 0.5)
    k_out, v_out, idx, scores = nat.keydiff_compress(k, v, n_kept, return_indices=True, return_scores=True)
    assert torch.equal(k_out, _gather_dev(k, idx)) and torch.equal(v_out, _gather_dev(v, idx))
    _assert_topk_of_own_scores(scores, idx, n_kept, slice(0, 0))
    # device-side fp32 evaluation of the formula
    kf = k.float()
    kn = kf.norm(dim=-1, keepdim=True)
    anchor = (kf / kn.clamp_min(1e-12)).mean(dim=2, keepdim=True)
    hi = -((kf * anchor).sum(-1) / kn.squeeze(-1).clamp_min(1e-8) / anchor.norm(dim=-1).clamp_min(1e-8))
    assert (scores.float() - hi).abs().max().item() <= 2.0 ** -8
    # determinism: the anchor reduction has a fixed order
    again = nat.keydiff_score(k)
    assert torch.equal(again, scores)
