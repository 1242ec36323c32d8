"""Every C-ABI entry point on caches, outputs and scratch that lie past the 2 GiB and 4 GiB byte offsets.

The ABI takes 64-bit element strides and promises arbitrary outer strides (include/kvpress_b200.h, Conventions), and
the caches it serves are often larger than 2^31 bytes: one Llama-3-8B layer at 128k tokens and batch 8 is 2 GiB of K
and 2 GiB of V. A 32-bit offset anywhere in the address code (TMA maps, pointer arithmetic of the score kernels, the
select / compact copies, workspace and score rows) passes every small test and corrupts such batches. Here:

* the arena: one device allocation of 2^32 + 2^26 bytes, filled once with 0xFF (NaN in bf16 and fp16). Parts A and B
  build their large inputs as views of it; each case writes its seeded inputs into its own views before its calls.
* Part A, far inputs: small problems, [1, 3, S, D] (the offset carried by the head stride) and [3, 1, S, D] (by the
  batch stride), whose (b, h) rows 1 and 2 hold arena bytes 2^31 and 2^32 strictly inside them. Row layouts:
  "interleaved" position rows [K | V] (row stride 2D, both K and V on the boundaries), and "split" dense rows (row
  stride D) with each (b, h) block [K rows | V rows] ("split_k", K on the boundaries) or [V rows | K rows] ("split_v"):
  a V block that trails its K block by a whole row span cannot hold both boundaries with row 0 at offset 0. Caller
  scores ride the same boundaries through their (b, h) strides, with K and V in ordinary memory ("scores").
  Bars: 1. every output bitwise equals the same call on the same view rebuilt in a small buffer (same row stride,
  smaller outer strides, so the same code path); 2. the scores meet the float64 bar of their scorer (tests/
  gpu_support.py, tests/merging_backend.py; LagKV and CUR are held to bar 1); 3. compress outputs are the canonical
  lowest-index-ties top-k of the call's own scores and exact gathers of the far views, rerotated keys admissible.
* Part B, outputs past 2^31 bytes: K_out and V_out of 2.15 GB each from every compaction writer (select + compact,
  its rerotating copy, Streaming, Knorm's two kernels and its cluster kernel's own compaction, Merging's merge with
  2.5 GB of scratch), checked row by row.
* Part C, scores and workspace past 2^31 bytes: one [1, 1, S, D] row expanded (zero strides) to 8192 rows, so the
  scores and the workspace's key array pass 2^31 bytes while K stays at 32 MiB; every row must equal the single-row
  call bitwise. Then zero-stride caches through the tensor-core scorers against float64.
The CPU tests check that every compute entry point has a Part A case, that every placement really straddles the
boundaries and that each part's computed peak of device memory fits 12 GiB. A GPU test skips only when the device
reports less free memory than its part needs.
"""
import gc
import math
import re
import zlib
from pathlib import Path

import pytest
import torch

from oracle import press_oracle as O
from tests import merging_backend as MB
from tests.conftest import ulp16_diff
from tests.gpu_support import (_forced_head, _forced_tail, _gather, _native, _same, assert_compress,
                               assert_keydiff_vs_ref, assert_rerotated, assert_vs_ref64, ckv_assert_scores, ea_ref64,
                               kd_chain, keydiff_error_bound, keydiff_ref64, knorm_ref64, nca_error_bound, oa_ref64,
                               rope_inv_freq, snap_ref64, ulp_at)
from tests import non_causal_attention_backend as NB

gpu = pytest.mark.gpu
DEV = "cuda:0"
HEADER = Path(__file__).resolve().parent.parent / "include" / "kvpress_b200.h"
TWO31, TWO32 = 1 << 31, 1 << 32
ARENA_BYTES = TWO32 + (1 << 26)
MEMORY_LIMIT = 12 << 30
BF16, FP16 = torch.bfloat16, torch.float16


# --------------------------------------------------------------------------------------------------
# the arena
# --------------------------------------------------------------------------------------------------
class _Arena:
    """The one 2^32 + 2^26-byte allocation of Parts A and B, made on first use and released before Part C."""
    buf = None

    @classmethod
    def get(cls) -> torch.Tensor:
        if cls.buf is None:
            cls.buf = torch.full((ARENA_BYTES,), 0xFF, dtype=torch.uint8, device=DEV)
        return cls.buf

    @classmethod
    def release(cls):
        cls.buf = None
        free_device_memory()


def free_device_memory():
    """Drop the wrappers' cached workspaces and torch's cached blocks, so that each large call starts from what is
    live."""
    _native()._WS_CACHE.clear()
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def require_memory(need: int, part: str):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    free, _ = torch.cuda.mem_get_info()
    held = 0 if _Arena.buf is None else ARENA_BYTES
    if free + held < need:
        pytest.skip(f"{part} needs {need} bytes of device memory, {free + held} are free")


def view16(dtype, shape, strides, offset=0, storage=None):
    """A 16-bit as_strided view of `storage` (default: the arena) at element `offset`."""
    base = (_Arena.get() if storage is None else storage).view(dtype)
    return torch.as_strided(base, shape, strides, offset)


# --------------------------------------------------------------------------------------------------
# Part A geometry
# --------------------------------------------------------------------------------------------------
LAYOUTS = ("interleaved", "split_k", "split_v")
CARRIES = ("head", "batch")


def shape_of(carry: str, S: int, D: int):
    return (1, 3, S, D) if carry == "head" else (3, 1, S, D)


def block(layout: str, S: int, D: int):
    """(row stride, element offset of K, of V, within one (b, h) block; the lead tensor's offset, its span in
    elements). One block holds 2 S D elements in every layout."""
    if layout == "interleaved":
        return 2 * D, 0, D, D, (S - 1) * 2 * D + D  # V leads: its boundary rows hold K's too
    if layout == "split_k":
        return D, 0, S * D, 0, S * D
    return D, S * D, 0, 0, S * D  # split_v: V first


def straddle_stride(lead: int, span: int) -> int:
    """Element stride X of rows at 0, X, 2X such that the span elements starting `lead` elements into row 1 hold byte
    2^31 strictly inside them and those of row 2 byte 2^32: row 1 starts h = span / 4 bytes (16-byte multiple) before
    2^31 - 2 lead, so row 2 starts 2 (lead + h) bytes before 2^32, which is inside its span."""
    h = (2 * span // 4) // 16 * 16
    return (TWO31 - 2 * lead - h) // 2


def outer_strides(carry: str, X: int):
    return (3 * X, X) if carry == "head" else (X, X)


def far_kv(layout, carry, S, D, dtype):
    """K and V views of the arena for a Part A case."""
    rs, ko, vo, lead, span = block(layout, S, D)
    X = straddle_stride(lead, span)
    sb, sh = outer_strides(carry, X)
    shape = shape_of(carry, S, D)
    return view16(dtype, shape, (sb, sh, rs, 1), ko), view16(dtype, shape, (sb, sh, rs, 1), vo)


def near_kv(layout, carry, S, D, dtype):
    """The same views rebuilt in a small NaN-filled buffer: same row stride, outer strides one block."""
    rs, ko, vo, _, _ = block(layout, S, D)
    X = 2 * S * D
    buf = torch.full((3 * X * 2,), 0xFF, dtype=torch.uint8, device=DEV)
    sb, sh = outer_strides(carry, X)
    shape = shape_of(carry, S, D)
    return (view16(dtype, shape, (sb, sh, rs, 1), ko, buf), view16(dtype, shape, (sb, sh, rs, 1), vo, buf))


def far_scores(carry, S, dtype):
    X = straddle_stride(0, S)
    sb, sh = outer_strides(carry, X)
    B, H = shape_of(carry, S, 8)[:2]
    return torch.as_strided(_Arena.get().view(dtype), (B, H, S), (sb, sh, 1))


# --------------------------------------------------------------------------------------------------
# Part A: the calls of every entry point, and their float64 bars
# --------------------------------------------------------------------------------------------------
def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(g, *shape, scale=1.0):
    return scale * torch.randn(*shape, generator=g, device=DEV)


def n_kept_of(S):
    return (2 * S) // 5 + 1


def _knorm_first_path(first: int) -> int:
    return _native().load().kvp_debug_knorm_first_path(first)


def call_knorm(k, v, ex, sc):
    nat = _native()
    S, n = k.shape[2], n_kept_of(k.shape[2])
    outs = {"score": nat.knorm_score(k)}
    for first in (0, 1, 2):
        previous = _knorm_first_path(first)
        try:
            launches = nat.launches_per_compress(nat.make_problem(k, v, n), nat.SCORER_KNORM)
            want = (1 if S <= 4096 else 2) if first == 0 else first + 1
            assert launches == want, f"knorm first path {first}: {launches} launches, expected {want}"
            outs[f"path{first}"] = nat.knorm_compress(k, v, n, True, True)
        finally:
            _knorm_first_path(previous)
    return outs


def bar_knorm(k, v, ex, sc, outs, what):
    S, n = k.shape[2], n_kept_of(k.shape[2])
    none = torch.zeros(S, dtype=torch.bool)
    ref = knorm_ref64(k)
    assert_vs_ref64(outs["score"], ref, none, f"{what} score")
    for first in (0, 1, 2):
        k_out, v_out, idx, s = outs[f"path{first}"]
        assert_vs_ref64(s, ref, none, f"{what} path {first}")
        assert_compress(k, v, k_out, v_out, idx, s, n)


def call_streaming(k, v, ex, sc):
    return {"compress": _native().streaming_compress(k, v, n_kept_of(k.shape[2]), 4, return_indices=True)}


def bar_streaming(k, v, ex, sc, outs, what):
    S, n = k.shape[2], n_kept_of(k.shape[2])
    k_out, v_out, idx = outs["compress"]
    assert torch.equal(idx.long().cpu(), O.streaming_kept(S, n, 4).expand(idx.shape)), what
    assert torch.equal(k_out, _gather(k, idx)) and torch.equal(v_out, _gather(v, idx)), what


SNAP_W = 64


def inputs_snapkv(B, H, G, S, D, dtype, g):
    return {"q": _randn(g, B, H * G, SNAP_W, D, scale=1.5).to(dtype)}


def call_snapkv(k, v, ex, sc):
    nat, n = _native(), n_kept_of(k.shape[2])
    return {"score": nat.snapkv_score(k, ex["q"], SNAP_W, 5),
            "compress": nat.snapkv_compress(k, v, ex["q"], SNAP_W, 5, n, True, True)}


def bar_snapkv(k, v, ex, sc, outs, what):
    S = k.shape[2]
    forced = _forced_tail(S, SNAP_W)
    ref = snap_ref64(ex["q"], k, SNAP_W, 5)
    assert_vs_ref64(outs["score"], ref, forced, f"{what} score", ftz=True)
    _check_compress(k, v, outs, what)


def _check_compress(k, v, outs, what):
    k_out, v_out, idx, s = outs["compress"]
    assert _same(s, outs["score"]), f"{what}: compress scores differ from the score call"
    assert_compress(k, v, k_out, v_out, idx, s, n_kept_of(k.shape[2]))


def inputs_ea(B, H, G, S, D, dtype, g):
    a = _randn(g, B, H * G, D, D) / D ** 0.5
    return {"mu": _randn(g, B, H * G, D, scale=0.5).to(dtype), "cov": (a @ a.transpose(-1, -2)).to(dtype)}


def call_ea(k, v, ex, sc):
    nat, n = _native(), n_kept_of(k.shape[2])
    return {"score": nat.expected_attention_score(k, v, ex["mu"], ex["cov"], 0.01, 4, True),
            "compress": nat.expected_attention_compress(k, v, ex["mu"], ex["cov"], 0.01, 4, True, n, True, True)}


def bar_ea(k, v, ex, sc, outs, what):
    ref = ea_ref64(k, v, ex["mu"], ex["cov"], 0.01, 4, True)
    assert_vs_ref64(outs["score"], ref, _forced_head(k.shape[2], 4), f"{what} score")
    _check_compress(k, v, outs, what)


def call_keydiff(k, v, ex, sc):
    nat, n = _native(), n_kept_of(k.shape[2])
    return {"score": nat.keydiff_score(k), "compress": nat.keydiff_compress(k, v, n, True, True)}


def bar_keydiff(k, v, ex, sc, outs, what):
    S, D = k.shape[2:]
    assert_keydiff_vs_ref(outs["score"], keydiff_ref64(k), keydiff_error_bound(k, kd_chain(S, D)), f"{what} score")
    _check_compress(k, v, outs, what)


CKV_EPS = 1e-3


def inputs_ckv(B, H, G, S, D, dtype, g):
    return {"wo": (_randn(g, 256, H * G * D) / math.sqrt(D)).to(dtype),
            "scores": torch.rand((B, H, S), generator=g, device=DEV).to(dtype)}


def call_ckv(k, v, ex, sc):
    nat, n = _native(), n_kept_of(k.shape[2])
    n_first = n // 4
    return {"score": nat.criticalkv_score(sc, v, ex["wo"], CKV_EPS, n_first),
            "compress": nat.criticalkv_compress(sc, k, v, ex["wo"], CKV_EPS, n_first, n, True, True)}


def bar_ckv(k, v, ex, sc, outs, what):
    n_first = n_kept_of(k.shape[2]) // 4
    ckv_assert_scores(outs["score"], sc, v, ex["wo"], CKV_EPS, n_first, f"{what} score")
    _check_compress(k, v, outs, what)


OA_NQ = 100


def inputs_oa(B, H, G, S, D, dtype, g):
    return {"q": _randn(g, B, H * G, OA_NQ, D, scale=1.5).to(dtype)}


def call_oa(k, v, ex, sc):
    nat, n = _native(), n_kept_of(k.shape[2])
    s = k.shape[3] ** -0.5
    return {"score": nat.observed_attention_score(k, ex["q"], s),
            "compress": nat.observed_attention_compress(k, v, ex["q"], s, n, True, True)}


def bar_oa(k, v, ex, sc, outs, what):
    S, D = k.shape[2:]
    ref = oa_ref64(k, ex["q"], D ** -0.5)
    assert_vs_ref64(outs["score"], ref, torch.zeros(S, dtype=torch.bool), f"{what} score", ftz=True)
    _check_compress(k, v, outs, what)


def inputs_nca(B, H, G, S, D, dtype, g):
    return {"q": _randn(g, B, H * G, S, D, scale=6 ** 0.5 / D ** 0.25).to(dtype), "cs": 128 if D == 64 else 256}


def nca_kv(B, H, S, D, dtype, g):
    """Keys of the logit spread of tests/gpu_support.nca_inputs and value rows with log-normal norms."""
    k = _randn(g, B, H, S, D, scale=6 ** 0.5 / D ** 0.25).to(dtype)
    v = (torch.exp(0.7 * _randn(g, B, H, S, 1)) * _randn(g, B, H, S, D)).to(dtype)
    return k, v


def call_nca(k, v, ex, sc):
    nat, n = _native(), n_kept_of(k.shape[2])
    return {"score": nat.non_causal_attention_score(k, v, ex["q"], ex["cs"]),
            "compress": nat.non_causal_attention_compress(k, v, ex["q"], ex["cs"], n, True, True)}


def bar_nca(k, v, ex, sc, outs, what):
    cs, q = ex["cs"], ex["q"]
    B, H, S, D = k.shape
    block_ = max(1, (1 << 25) // (B * q.shape[1] * cs * cs))
    x64, tau = NB.non_causal_attention_parts64(k, v, q, cs, block=block_, with_bound=True)
    z64 = NB.zscore64(x64)
    E = nca_error_bound(x64, tau, z64, cs, D, q.shape[1] // H)
    got = outs["score"]
    near = (got.double() - z64).abs() <= ulp_at(z64, got.dtype) / 2 + E
    ok = (ulp16_diff(got, z64.to(got.dtype)) <= 1) | near
    assert ok.all(), f"{what}: {int((~ok).sum())} scores beyond 1 ulp and beyond the error bound of the fp64 z-score"
    _check_compress(k, v, outs, what)


def call_lagkv(k, v, ex, sc):
    nat, n = _native(), n_kept_of(k.shape[2])
    return {"score": nat.lagkv_score(k, v, 4, 64, False),
            "compress": nat.lagkv_compress(k, v, 4, 64, False, n, True, True)}


def bar_scores_only(k, v, ex, sc, outs, what):
    _check_compress(k, v, outs, what)


def inputs_cur(B, H, G, S, D, dtype, g):
    return {"G": _randn(g, D, 8) / 8 ** 0.5}


def call_cur(k, v, ex, sc):
    nat, n = _native(), n_kept_of(k.shape[2])
    return {"score": nat.cur_score(k, v, 2, "kv_avg", 16, ex["G"]),
            "compress": nat.cur_compress(k, v, 2, "kv_avg", 16, ex["G"], n, True, True)}


def inputs_scores(B, H, G, S, D, dtype, g):
    return {"scores": _randn(g, B, H, S).to(dtype), "inv_freq": rope_inv_freq("theta500000", D).to(DEV)}


def call_generic(k, v, ex, sc):
    nat, n = _native(), n_kept_of(k.shape[2])
    return {"compress": nat.scores_compress(sc, k, v, n, True), "select": nat.scores_select(sc, n),
            "rerotate": nat.scores_compress_rerotate(sc, k, v, n, ex["inv_freq"], True)}


def bar_generic(k, v, ex, sc, outs, what):
    n = n_kept_of(k.shape[2])
    k_out, v_out, idx = outs["compress"]
    assert_compress(k, v, k_out, v_out, idx, sc, n)
    assert torch.equal(outs["select"], idx), f"{what}: scores_select differs from scores_compress"
    assert_rerotated(k, v, sc, n, ex["inv_freq"], outs["rerotate"], what)


MERGE_THR, MERGE_FRAC = 0.0, 1.0


def call_merging(k, v, ex, sc):
    nat, n = _native(), n_kept_of(k.shape[2])
    compress = nat.merging_compress(sc, k, v, MERGE_THR, MERGE_FRAC, n, True, True)
    return {"compress": compress, "merge": nat.merging_merge(k, v, compress[2], MERGE_THR, MERGE_FRAC, True)}


def assert_merge64(k, v, kept, v_out, target, sim, what):
    """The plan against float64 cosine similarities (targets may differ only where the best two are within 1e-5),
    the values against the float64 merge on the kernel's own plan."""
    t64, max64 = MB.plan64(k, kept)
    assert ((sim.double() - max64).abs() <= 1e-5).all(), f"{what}: max_sim beyond 1e-5 of float64"
    at = MB.similarities64(k, kept).gather(-1, target.long().unsqueeze(-1)).squeeze(-1)
    assert ((target.long() == t64) | (at >= max64 - 1e-5)).all(), f"{what}: a target is not the float64 argmax"
    ok = MB.gate(sim, MERGE_THR, MERGE_FRAC)
    v64 = MB.merged_values64(v, kept, target, sim.double(), ok)
    scale = v.double().abs().amax()
    bad = (v_out.double() - v64).abs() > ulp_at(v64, v.dtype) + 2.0 ** -16 * scale
    assert not bad.any(), f"{what}: {int(bad.sum())} merged values beyond 1 ulp of float64"


def bar_merging(k, v, ex, sc, outs, what):
    n = n_kept_of(k.shape[2])
    k_out, v_out, idx, target, sim = outs["compress"]
    assert torch.equal(idx.long().cpu(), O.select_lowest_index_ties(sc.cpu(), n)), f"{what}: not the canonical set"
    assert torch.equal(k_out, _gather(k, idx)), f"{what}: K' is not an exact gather"
    if k.shape[2] <= 4096:  # the float64 similarities of one 32k row take 2 GB: there bar 1 holds alone
        assert_merge64(k, v, idx, v_out, target, sim, f"{what} compress")
    m_out, m_target, m_sim = outs["merge"]
    assert _same(m_out, v_out) and torch.equal(m_target, target) and torch.equal(m_sim, sim), \
        f"{what}: merge differs from compress"


# family -> (entry points it calls, call, bar, extra inputs, takes caller scores, configs)
TC = [(BF16, 64, 1, 1000), (BF16, 128, 4, 1000), (FP16, 64, 4, 1000), (FP16, 128, 1, 1000), (BF16, 128, 1, 32768)]
CC = [(BF16, 32, 1, 1000), (FP16, 64, 1, 1000), (BF16, 128, 1, 1000), (FP16, 256, 1, 1000), (BF16, 128, 1, 32768)]
FAMILIES = {
    "knorm": (("kvp_knorm_score", "kvp_knorm_compress"), call_knorm, bar_knorm, None, False, CC),
    "streaming": (("kvp_streaming_compress",), call_streaming, bar_streaming, None, False,
                  [(BF16, 128, 1, 1000), (FP16, 64, 1, 1000), (BF16, 128, 1, 32768)]),
    "snapkv": (("kvp_snapkv_score", "kvp_snapkv_compress"), call_snapkv, bar_snapkv, inputs_snapkv, False, TC),
    "ea": (("kvp_expected_attention_score", "kvp_expected_attention_compress"), call_ea, bar_ea, inputs_ea, False, TC),
    "keydiff": (("kvp_keydiff_score", "kvp_keydiff_compress"), call_keydiff, bar_keydiff, None, False, CC),
    "criticalkv": (("kvp_criticalkv_score", "kvp_criticalkv_compress"), call_ckv, bar_ckv, inputs_ckv, True, TC),
    "observed_attention": (("kvp_observed_attention_score", "kvp_observed_attention_compress"), call_oa, bar_oa,
                           inputs_oa, False, TC),
    "non_causal_attention": (("kvp_non_causal_attention_score", "kvp_non_causal_attention_compress"), call_nca,
                             bar_nca, inputs_nca, False, TC),
    "lagkv": (("kvp_lagkv_score", "kvp_lagkv_compress"), call_lagkv, bar_scores_only, None, False, CC),
    "cur": (("kvp_cur_score", "kvp_cur_compress"), call_cur, bar_scores_only, inputs_cur, False, CC),
    "generic": (("kvp_scores_compress", "kvp_scores_select", "kvp_scores_compress_rerotate"), call_generic,
                bar_generic, inputs_scores, True, CC),
    "merging": (("kvp_merging_compress", "kvp_merging_merge"), call_merging, bar_merging, inputs_scores, True, CC),
}
# kvp_streaming_score reads no K: nothing of it lies far
EXEMPT = {"kvp_streaming_score"}


def _cfg_id(cfg):
    dtype, D, G, S = cfg
    return f"{'bf16' if dtype == BF16 else 'fp16'}-D{D}-G{G}-S{S}"


def part_a_cases():
    out = []
    for fam, (_, _, _, _, caller, cfgs) in FAMILIES.items():
        places = [(lay, c) for lay in LAYOUTS for c in CARRIES] + ([("scores", c) for c in CARRIES] if caller else [])
        for cfg in cfgs:
            for lay, carry in places:
                out.append(pytest.param(fam, cfg, lay, carry, id=f"{fam}-{_cfg_id(cfg)}-{lay}-{carry}"))
    return out


def _flat(outs):
    for key in sorted(outs):
        val = outs[key]
        for i, t in enumerate(val if isinstance(val, tuple) else (val,)):
            yield f"{key}[{i}]", t


def part_a_need(cfg) -> int:
    _, D, G, S = cfg
    return ARENA_BYTES + (256 << 20) + 64 * 3 * S * D * max(G, 1)


@gpu
@pytest.mark.parametrize("fam, cfg, layout, carry", part_a_cases())
def test_far_inputs(fam, cfg, layout, carry):
    require_memory(part_a_need(cfg), "Part A")
    nat = _native()
    _, call, bar, make_inputs, caller, _ = FAMILIES[fam]
    dtype, D, G, S = cfg
    B, H = shape_of(carry, S, D)[:2]
    what = f"{fam} {_cfg_id(cfg)} {layout} {carry}"
    g = _gen(zlib.crc32(what.encode()))
    if fam == "non_causal_attention":
        kd, vd = nca_kv(B, H, S, D, dtype, g)
    else:
        scale = torch.exp(0.3 * _randn(g, B, H, S, 1))
        kd, vd = (scale * _randn(g, B, H, S, D)).to(dtype), _randn(g, B, H, S, D).to(dtype)
    ex = make_inputs(B, H, G, S, D, dtype, g) if make_inputs else {}
    near_sc = ex.get("scores")
    if layout == "scores":
        k_far = k_near = kd
        v_far = v_near = vd
        sc_far = far_scores(carry, S, dtype)
        sc_far.copy_(near_sc)
        assert sc_far.stride(-1) == 1, "far scores are consumed in place"
    else:
        k_far, v_far = far_kv(layout, carry, S, D, dtype)
        k_near, v_near = near_kv(layout, carry, S, D, dtype)
        for t, d in ((k_far, kd), (v_far, vd), (k_near, kd), (v_near, vd)):
            t.copy_(d)
        sc_far = near_sc
    for t in (k_far, v_far):
        assert nat._rows_ok(t), "the wrapper would hand a compact copy to the C ABI"
    far = call(k_far, v_far, ex, sc_far)
    near = call(k_near, v_near, ex, near_sc)
    torch.cuda.synchronize()
    for (name, a), (_, b) in zip(_flat(far), _flat(near)):
        assert _same(a, b), f"{what}: {name} differs from the same call in a small buffer"
    bar(k_far, v_far, ex, sc_far, far, what)


# --------------------------------------------------------------------------------------------------
# Part B: K_out / V_out past 2^31 bytes
# --------------------------------------------------------------------------------------------------
LONG = (8, 8, 131584, 128)  # interleaved [K | V] rows over the whole arena
LONG_KEPT = 131328
SHORT = (16, 129, 4096, 128)  # split dense [K rows | V rows] blocks
SHORT_KEPT = 4088


def long_kv(dtype=BF16):
    B, H, S, D = LONG
    st = (H * S * 2 * D, S * 2 * D, 2 * D, 1)
    return view16(dtype, LONG, st, 0), view16(dtype, LONG, st, D)


def short_kv(dtype=BF16):
    B, H, S, D = SHORT
    st = (H * 2 * S * D, 2 * S * D, D, 1)
    return view16(dtype, SHORT, st, 0), view16(dtype, SHORT, st, S * D)


def out_bytes(shape, n_kept):
    B, H, _, D = shape
    return B * H * n_kept * D * 2


def ws_bytes(shape, n_kept, scorer) -> int:
    """kvp_workspace_bytes of a bf16 [B, H, S, D] problem (the strides do not enter it)."""
    nat = _native()
    p = nat.KvpProblem()
    (p.B, p.Hkv, p.S, p.D), p.Hq, p.n_kept, p.dtype = shape, shape[1], n_kept, 0
    return nat.workspace_bytes(p, scorer)


def part_b_peak() -> int:
    nat = _native()
    B, H, S, D = LONG
    small = B * H * S * 2 * 4 + B * H * LONG_KEPT * 4 * 2  # caller scores (+ a copy), idx, kept
    long_calls = [2 * out_bytes(LONG, LONG_KEPT) + ws_bytes(LONG, LONG_KEPT, s)
                  for s in (nat.SCORER_GENERIC, nat.SCORER_KNORM)]
    long_calls.append(out_bytes(LONG, LONG_KEPT) + ws_bytes(LONG, LONG_KEPT, nat.SCORER_MERGING))
    short = 2 * out_bytes(SHORT, SHORT_KEPT) + SHORT[0] * SHORT[1] * SHORT[2] * 2
    # + 1 GiB for the checks' per-row and per-batch temporaries
    return ARENA_BYTES + small + max(max(long_calls), short) + (1 << 30)


_LONG = {}  # the inputs of the long-row cases, written once; dropped with the arena before Part C


@pytest.fixture
def long_rows():
    """Seeded K / V filling the whole arena as the LONG interleaved cache, and caller scores with planted ties."""
    require_memory(part_b_peak(), "Part B")
    if "kv" not in _LONG:
        print(f"[measured] Part A peak {torch.cuda.max_memory_allocated()} bytes")  # Part A runs first
        _LONG["kv"] = _long_inputs()
    return _LONG["kv"]


def _long_inputs():
    k, v = long_kv()
    B, H, S, D = LONG
    g = _gen(2024)
    for b in range(B):  # one batch (512 MiB of K and V) at a time
        k[b].copy_(_randn(g, H, S, D).to(BF16))
        v[b].copy_(_randn(g, H, S, D).to(BF16))
    sc = _randn(g, B, H, S).to(BF16)
    # ties planted across each row's threshold: 600 positions of one value, straddling rank n_kept
    thr = sc.float().sort(dim=-1, descending=True).values[..., LONG_KEPT - 1:LONG_KEPT]
    pos = torch.randperm(S, generator=torch.Generator().manual_seed(3))[:600].to(DEV)
    sc[..., pos] = thr.to(BF16).expand(B, H, 600)
    return k, v, sc


def check_rows(k, v, idx, k_out, v_out, want_idx, what):
    """One (b, h) row at a time, so that no second 2 GiB tensor is made: idx as wanted, K_out / V_out rows the exact
    gathers of the far inputs."""
    B, H = k.shape[:2]
    for b in range(B):
        for h in range(H):
            i = idx[b, h].long()
            assert torch.equal(i.cpu(), want_idx(b, h)), f"{what}: row ({b}, {h}) keeps the wrong positions"
            assert _same(k_out[b, h], k[b, h].index_select(0, i)), f"{what}: K_out row ({b}, {h})"
            assert _same(v_out[b, h], v[b, h].index_select(0, i)), f"{what}: V_out row ({b}, {h})"


def canonical(sc, n):
    return lambda b, h: O.select_lowest_index_ties(sc[b, h][None].cpu(), n)[0]


@gpu
def test_long_rows_scores_compress(long_rows):
    k, v, sc = long_rows
    free_device_memory()
    torch.cuda.reset_peak_memory_stats()
    k_out, v_out, idx = _native().scores_compress(sc, k, v, LONG_KEPT, True)
    torch.cuda.synchronize()
    assert k_out.numel() * 2 > TWO31 and k.storage_offset() == 0
    check_rows(k, v, idx, k_out, v_out, canonical(sc, LONG_KEPT), "scores_compress")
    print(f"[measured] Part B scores_compress peak {torch.cuda.max_memory_allocated()} bytes")


@gpu
def test_long_rows_knorm_two_kernels(long_rows):
    k, v, _ = long_rows
    nat = _native()
    free_device_memory()
    assert nat.launches_per_compress(nat.make_problem(k, v, LONG_KEPT), nat.SCORER_KNORM) == 3
    k_out, v_out, idx, sc = nat.knorm_compress(k, v, LONG_KEPT, True, True)
    torch.cuda.synchronize()
    check_rows(k, v, idx, k_out, v_out, canonical(sc, LONG_KEPT), "knorm_compress two kernels")
    B, H = LONG[:2]
    for b, h in ((0, 0), (B - 1, H - 1)):
        assert_vs_ref64(sc[b:b + 1, h:h + 1], knorm_ref64(k[b:b + 1, h:h + 1]), torch.zeros(LONG[2], dtype=torch.bool),
                        f"knorm long row ({b}, {h})")


@gpu
def test_long_rows_streaming(long_rows):
    k, v, _ = long_rows
    free_device_memory()
    k_out, v_out, idx = _native().streaming_compress(k, v, LONG_KEPT, 4, return_indices=True)
    torch.cuda.synchronize()
    want = O.streaming_kept(LONG[2], LONG_KEPT, 4)
    check_rows(k, v, idx, k_out, v_out, lambda b, h: want, "streaming_compress")


@gpu
def test_long_rows_rerotate(long_rows):
    k, v, sc = long_rows
    free_device_memory()
    inv = rope_inv_freq("theta500000", LONG[3]).to(DEV)
    k_out, v_out, idx = _native().scores_compress_rerotate(sc, k, v, LONG_KEPT, inv, True)
    torch.cuda.synchronize()
    B, H = LONG[:2]
    for b in range(B):
        for h in range(H):
            r = (slice(b, b + 1), slice(h, h + 1))
            assert_rerotated(k[r], v[r], sc[r], LONG_KEPT, inv, (k_out[r], v_out[r], idx[r]), f"rerotate ({b}, {h})")


@gpu
def test_long_rows_merge(long_rows):
    """merging_merge over 64 rows with 2.5 GB of scratch: the first and last rows, and the row whose output span holds
    byte 2^31, are bitwise equal to the same row merged alone (a row's result does not depend on its batch)."""
    k, v, sc = long_rows
    nat = _native()
    free_device_memory()
    torch.cuda.reset_peak_memory_stats()
    kept = nat.scores_select(sc, LONG_KEPT)
    v_out, target, sim = nat.merging_merge(k, v, kept, 0.0, 1.0, True)
    torch.cuda.synchronize()
    B, H, S, D = LONG
    row_bytes = LONG_KEPT * D * 2
    rows = sorted({0, TWO31 // row_bytes, B * H - 1})
    assert TWO31 // row_bytes * row_bytes < TWO31 < (TWO31 // row_bytes + 1) * row_bytes
    print(f"[measured] Part B merge peak {torch.cuda.max_memory_allocated()} bytes")
    for r in rows:
        b, h = divmod(r, H)
        s = (slice(b, b + 1), slice(h, h + 1))
        alone = nat.merging_merge(k[s], v[s], kept[s], 0.0, 1.0, True)
        torch.cuda.synchronize()
        assert _same(v_out[s], alone[0]), f"merged row ({b}, {h}) depends on the batch"
        assert torch.equal(target[s], alone[1]) and torch.equal(sim[s], alone[2]), f"plan of row ({b}, {h})"


@gpu
def test_short_rows_knorm_cluster():
    """The cluster kernel's own compaction (bulk row copies of dense rows) writing 2.16 GB per output."""
    require_memory(part_b_peak(), "Part B")
    nat = _native()
    _LONG.clear()  # the short rows overwrite the arena
    free_device_memory()
    torch.cuda.reset_peak_memory_stats()
    k, v = short_kv()
    B, H, S, D = SHORT
    g = _gen(77)
    for b in range(B):
        k[b].copy_((torch.exp(0.3 * _randn(g, H, S, 1)) * _randn(g, H, S, D)).to(BF16))
        v[b].copy_(_randn(g, H, S, D).to(BF16))
    assert nat._rows_ok(k) and nat._rows_ok(v)
    assert nat.launches_per_compress(nat.make_problem(k, v, SHORT_KEPT), nat.SCORER_KNORM) == 1
    k_out, v_out, idx, sc = nat.knorm_compress(k, v, SHORT_KEPT, True, True)
    torch.cuda.synchronize()
    assert k_out.numel() * 2 > TWO31
    want = O.select_lowest_index_ties(sc.cpu(), SHORT_KEPT)
    assert torch.equal(idx.long().cpu(), want), "knorm cluster: not the canonical selection of its scores"
    for b in range(B):  # one batch (135 MB of each output) at a time
        assert _same(k_out[b], _gather(k[b:b + 1], idx[b:b + 1])[0]), f"knorm cluster: K_out batch {b}"
        assert _same(v_out[b], _gather(v[b:b + 1], idx[b:b + 1])[0]), f"knorm cluster: V_out batch {b}"
    ref = knorm_ref64(k[:1])
    assert_vs_ref64(sc[:1], ref, torch.zeros(S, dtype=torch.bool), "knorm cluster batch 0")
    print(f"[measured] Part B short rows peak {torch.cuda.max_memory_allocated()} bytes")


# --------------------------------------------------------------------------------------------------
# Part C: scores and workspace past 2^31 bytes
# --------------------------------------------------------------------------------------------------
WIDE = (64, 128, 131328, 128)
WIDE_KEPT = 64
PART_C_NAMES = ["knorm_score", "knorm_compress", "keydiff_score", "keydiff_compress", "lagkv_score", "lagkv_compress",
                "streaming_score", "streaming_compress", "scores_select", "scores_compress"]


def part_c_calls():
    """(name, scorer, scores bytes written or read, output bytes) of every Part C call."""
    nat = _native()
    B, H, S, D = WIDE
    sc, outs = B * H * S * 2, 2 * out_bytes(WIDE, WIDE_KEPT) + B * H * WIDE_KEPT * 4
    return [("knorm_score", None, sc, 0), ("knorm_compress", nat.SCORER_KNORM, sc, outs),
            ("keydiff_score", nat.SCORER_KEYDIFF, sc, 0), ("keydiff_compress", nat.SCORER_KEYDIFF, sc, outs),
            ("lagkv_score", nat.SCORER_LAGKV, sc, 0), ("lagkv_compress", nat.SCORER_LAGKV, sc, outs),
            ("streaming_score", None, sc, 0), ("streaming_compress", None, 0, outs),
            ("scores_select", nat.SCORER_GENERIC, sc, B * H * WIDE_KEPT * 4),
            ("scores_compress", nat.SCORER_GENERIC, sc, outs)]


def part_c_peak() -> int:
    return max(s + o + (0 if w is None else ws_bytes(WIDE, WIDE_KEPT, w)) for _, w, s, o in part_c_calls()) \
        + (512 << 20)


def wide_kv(dtype=BF16):
    B, H, S, D = WIDE
    g = _gen(4242)
    k1 = (torch.exp(0.3 * _randn(g, 1, 1, S, 1)) * _randn(g, 1, 1, S, D)).to(dtype)
    v1 = _randn(g, 1, 1, S, D).to(dtype)
    return k1, v1, k1.expand(WIDE), v1.expand(WIDE)


def assert_rows_equal(wide, one, what, rows=512):
    """Every (b, h) row of `wide` [B, H, ...] is bitwise `one` [1, 1, ...], compared a chunk of rows at a time."""
    flat = wide.reshape(-1, *wide.shape[2:])
    o = one.reshape(1, *one.shape[2:])
    if o.dtype in (BF16, FP16):
        flat, o = flat.view(torch.int16), o.view(torch.int16)
    for r0 in range(0, flat.shape[0], rows):
        bad = (flat[r0:r0 + rows] != o).flatten(1).any(1)
        assert not bad.any(), f"{what}: row {r0 + int(bad.nonzero()[0])} differs from the single-row call"


def _wide_call(name, k, v, sc=None):
    nat = _native()
    return {"knorm_score": lambda: (nat.knorm_score(k),),
            "knorm_compress": lambda: nat.knorm_compress(k, v, WIDE_KEPT, True, True),
            "keydiff_score": lambda: (nat.keydiff_score(k),),
            "keydiff_compress": lambda: nat.keydiff_compress(k, v, WIDE_KEPT, True, True),
            "lagkv_score": lambda: (nat.lagkv_score(k, v, 4, 64, False),),
            "lagkv_compress": lambda: nat.lagkv_compress(k, v, 4, 64, False, WIDE_KEPT, True, True),
            "streaming_score": lambda: (nat.streaming_score(k, WIDE_KEPT, 4),),
            "streaming_compress": lambda: nat.streaming_compress(k, v, WIDE_KEPT, 4, True),
            "scores_select": lambda: (nat.scores_select(sc, WIDE_KEPT),),
            "scores_compress": lambda: nat.scores_compress(sc, k, v, WIDE_KEPT, True)}[name]()


@pytest.fixture(scope="module")
def wide_rows():
    require_memory(part_c_peak(), "Part C")  # counts the arena as free: it is released here
    _LONG.clear()
    _Arena.release()
    return wide_kv()


@gpu
@pytest.mark.parametrize("name", PART_C_NAMES)
def test_wide_rows_match_one_row(name, wide_rows):
    k1, v1, k, v = wide_rows
    nat = _native()
    assert nat._rows_ok(k) and k.stride(0) == k.stride(1) == 0
    free_device_memory()
    sc = sc1 = None
    if name.startswith("scores_"):
        sc1 = _randn(_gen(9), 1, 1, WIDE[2]).to(BF16)
        sc = sc1.expand(WIDE[:3]).contiguous()  # a 2 GiB caller score tensor
    one = _wide_call(name, k1, v1, sc1)
    torch.cuda.reset_peak_memory_stats()
    got = _wide_call(name, k, v, sc)
    torch.cuda.synchronize()
    print(f"[measured] Part C {name} peak {torch.cuda.max_memory_allocated()} bytes")
    for i, (a, b) in enumerate(zip(got, one)):
        if a is not None:
            assert_rows_equal(a, b, f"{name} output {i}")
    del got, sc


# zero-stride caches through the tensor-core scorers, at small shapes, against float64
@gpu
@pytest.mark.parametrize("fam", ["snapkv", "ea", "criticalkv", "observed_attention", "non_causal_attention"])
def test_zero_stride_tensor_core_scorers(fam):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    _, call, bar, make_inputs, _, _ = FAMILIES[fam]
    dtype, D, G, S = BF16, 128, 2, 1000
    B, H = 2, 3
    g = _gen(5)
    if fam == "non_causal_attention":
        k1, v1 = nca_kv(1, 1, S, D, dtype, g)
    else:
        k1, v1 = _randn(g, 1, 1, S, D).to(dtype), _randn(g, 1, 1, S, D).to(dtype)
    k, v = k1.expand(B, H, S, D), v1.expand(B, H, S, D)
    assert _native()._rows_ok(k) and k.stride(1) == 0
    ex = make_inputs(B, H, G, S, D, dtype, g)
    sc = ex.get("scores")
    outs = call(k, v, ex, sc)
    torch.cuda.synchronize()
    bar(k, v, ex, sc, outs, f"{fam} zero strides")
    dense = call(k.contiguous(), v.contiguous(), ex, sc)
    torch.cuda.synchronize()
    for (name, a), (_, b) in zip(_flat(outs), _flat(dense)):
        assert _same(a, b), f"{fam}: {name} of the zero-stride cache differs from its dense copy"


# --------------------------------------------------------------------------------------------------
# CPU: coverage, placement, memory plan
# --------------------------------------------------------------------------------------------------
NOT_COMPUTE = re.compile(r"kvp_(abi_version|status_string|last_cuda_error|workspace_bytes|workspace_check|"
                         r"launches_per_compress|debug_\w+)$")
# each compaction writer of the library, and the Part B test that makes it write past 2^31 bytes
PART_B_WRITERS = {
    "select_compact copy_rows_kv (kvp_scores_compress)": test_long_rows_scores_compress,
    "select_compact copy_rows_kv (kvp_knorm_compress, two kernels)": test_long_rows_knorm_two_kernels,
    "streaming compaction (kvp_streaming_compress)": test_long_rows_streaming,
    "select_compact copy_rows_k_rerotated / copy_rows_single (kvp_scores_compress_rerotate)": test_long_rows_rerotate,
    "merging merge (kvp_merging_merge)": test_long_rows_merge,
    "knorm_cluster bulk-store compaction (kvp_knorm_compress, cluster)": test_short_rows_knorm_cluster,
}


def test_every_compute_entry_point_has_a_far_input_case():
    declared = set(re.findall(r"^int (kvp_\w+)\(", HEADER.read_text(), re.M))
    compute = {n for n in declared if not NOT_COMPUTE.match(n)} - EXEMPT
    covered = {e for fam in FAMILIES.values() for e in fam[0]}
    assert compute - covered == set(), f"entry points without a Part A case: {sorted(compute - covered)}"
    assert covered - declared == set(), f"Part A names entry points the header does not declare: {covered - declared}"
    assert {p.values[0] for p in part_a_cases()} == set(FAMILIES)
    assert all(callable(t) for t in PART_B_WRITERS.values()) and len(PART_B_WRITERS) == 6


def row_ranges(shape, strides, offset, width, esize=2):
    """Byte range [lo, hi) of every (b, h) row of a [B, H, S, ...] view: S rows of `width` elements."""
    B, H, S = shape[:3]
    out = []
    for b in range(B):
        for h in range(H):
            lo = (offset + b * strides[0] + h * strides[1]) * esize
            out.append((lo, lo + ((S - 1) * strides[2] + width) * esize))
    return out


def _straddles(ranges, byte):
    return any(lo < byte < hi for lo, hi in ranges)


def _check_view(shape, strides, offset, width, what):
    ranges = row_ranges(shape, strides, offset, width)
    assert min(lo for lo, _ in ranges) >= 0 and max(hi for _, hi in ranges) <= ARENA_BYTES, f"{what}: outside the arena"
    row_strides = strides[:3] if width > 1 else strides[:2]  # score rows are unit-stride
    assert offset * 2 % 16 == 0 and all(s % 8 == 0 for s in row_strides), f"{what}: rows not 16-byte aligned"
    return ranges


@pytest.mark.parametrize("fam, cfg, layout, carry", part_a_cases())
def test_part_a_placement(fam, cfg, layout, carry):
    _, D, _, S = cfg
    shape = shape_of(carry, S, D)
    if layout == "scores":
        X = straddle_stride(0, S)
        ranges = _check_view(shape[:3], (*outer_strides(carry, X), 1), 0, 1, "scores")
        rows = {"scores": ranges}
    else:
        rs, ko, vo, _, _ = block(layout, S, D)
        X = straddle_stride(*block(layout, S, D)[3:])
        st = (*outer_strides(carry, X), rs)
        rows = {"K": _check_view(shape, st, ko, D, "K"), "V": _check_view(shape, st, vo, D, "V")}
        k_lo = {lo for lo, _ in rows["K"]} | {lo for lo, _ in rows["V"]}
        assert min(k_lo) == 0, "row 0 sits at offset 0"
        if layout == "interleaved":
            assert rs == 2 * D and vo == ko + D
        else:
            assert rs == D and abs(vo - ko) == S * D
    want = {"K", "V"} if layout == "interleaved" else {"K"} if layout == "split_k" else {"V"} if layout == "split_v" \
        else {"scores"}
    for name in want:
        r = rows[name]
        assert r[1][0] < TWO31 < r[1][1] and r[2][0] < TWO32 < r[2][1], f"{name}: rows 1 and 2 miss the boundaries"
        assert not any(lo < TWO31 < hi for lo, hi in (r[0], r[2])) and not any(lo < TWO32 < hi for lo, hi in r[:2])


def test_part_b_placement():
    B, H, S, D = LONG
    ranges = _check_view(LONG, (H * S * 2 * D, S * 2 * D, 2 * D), D, D, "long V")
    assert _straddles(ranges, TWO31) and _straddles(ranges, TWO32)
    assert _straddles(_check_view(LONG, (H * S * 2 * D, S * 2 * D, 2 * D), 0, D, "long K"), TWO32)
    B, H, S, D = SHORT
    st = (H * 2 * S * D, 2 * S * D, D)
    assert max(hi for _, hi in _check_view(SHORT, st, 0, D, "short K")) > TWO32
    assert max(hi for _, hi in _check_view(SHORT, st, S * D, D, "short V")) > TWO32
    for shape, n in ((LONG, LONG_KEPT), (SHORT, SHORT_KEPT)):  # the output row that holds byte 2^31 straddles it
        assert out_bytes(shape, n) > TWO31
        out_rows = row_ranges((*shape[:2], n), (shape[1] * n * shape[3], n * shape[3], shape[3]), 0, shape[3])
        assert _straddles(out_rows, TWO31)
    assert S * D * 2 < (8 << 20)  # the short rows take the cluster path, the long ones select + compact's big rows
    assert LONG[2] * LONG[3] * 2 >= (8 << 20)


def test_part_c_placement():
    nat = _native()
    B, H, S, D = WIDE
    R, tile = B * H, 256
    n_tiles = -(-S // tile)
    a256 = lambda x: -(-x // 256) * 256  # noqa: E731
    keys_at = a256(R * 256 * 4) * 2 + a256((R * 3 + 64) * 4) + a256(R * n_tiles * 8)  # the carve order of api.cu
    keys_bytes = R * n_tiles * tile * 2
    assert keys_bytes > TWO31 and B * H * S * 2 > TWO31
    for _, w, _, _ in part_c_calls():
        if w is not None:
            assert ws_bytes(WIDE, WIDE_KEPT, w) >= keys_at + keys_bytes
    assert S * D * 2 <= (32 << 20) + S * D  # K stays one row of about 32 MiB
    assert nat.SCORER_GENERIC == 0


def test_memory_plan():
    part_a = max(part_a_need(cfg) for fam in FAMILIES.values() for cfg in fam[5])
    plan = {"A": part_a, "B": part_b_peak(), "C": part_c_peak()}
    print(f"[computed] device memory peaks: {plan}")
    assert all(v < MEMORY_LIMIT for v in plan.values()), plan
