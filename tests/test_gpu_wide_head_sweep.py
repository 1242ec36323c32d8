"""The torch GEMM score stage of kvpress_b200/wide_head_scores.py against float64 evaluations, at every kind of shape
the presses route to it, under both of torch's fp32 matmul precisions.

That module scores the shapes the sm_90a scorers do not instantiate (head_dim other than 64 / 128, more than 8 query
heads per kv head, SnapKV with G * window > 512, NonCausal chunk sizes other than 128 / 256) with fp32 GEMMs on the GPU,
and promises the kernels' contract: fp32 evaluation of the formula, rounded once to the cache dtype. Its scores then go
through the same selection kernels. Every GPU case runs under torch.backends.cuda.matmul.fp32_precision = "ieee" and
"tf32" (what torch.set_float32_matmul_precision("high") selects). Every GEMM operand is an exact 16-bit value and the
scales are applied to the fp32 products, so TF32 rounds nothing: both precisions must meet the same bars, and the
library must leave the setting as it found it.

Bars: the float64 references and bars of the kernel tests, unchanged.
- ExpectedAttention, SnapKV, ObservedAttention: tests/test_gpu_scorer_sweep.py (assert_vs_ref64). Within 1 ulp of the
  fp64 score rounded once, no row bias, forced positions equal round(max + 1). No ftz allowance: nothing here uses
  ex2.approx.ftz.
- CriticalKV: tests/test_gpu_criticalkv.py (assert_scores). 1 ulp, no row bias, the n_first best base scores of every
  row hold finfo.max.
- NonCausalAttention: |z - z64| <= ulp + 4 E_s, with E_s the a-priori fp32 error bound of
  tests/test_gpu_non_causal_attention.py; the factor 4 allows for cuBLAS's summation orders.
- After each score, native.scores_compress on it keeps the lowest-index-ties top-k and returns exact K / V gathers.

Cases, all on shapes the presses send here (a CPU test checks that, and that every condition of every routing predicate
is driven false):
- head_dim 32 / 80 / 96 / 160 / 256, and 64 / 128 with 9, 12 or 16 query heads per kv head;
- SnapKV: G * window 513 / 520 / 768 / 1024, window 1, S = window + 1, kernel sizes 1 / 3 / 7;
- ExpectedAttention: covariance on and off, use_vnorm x epsilon 0 / 1e-2, n_sink 0 / 1 / 4 / S - 1;
- CriticalKV: hidden 64 / 600 / 1000, n_first 0 / 1 / S / 3 / S;
- ObservedAttention: n_q 1 / 7 / S - 1 / S;
- NonCausal: chunk sizes 1 / 2 / 64 / 100 / 129 / 512, one larger than S, S one past a chunk;
- the slab and block loops crossed at their edges, through small `chunk` / `max_logits` arguments;
- one peaked case per softmax scorer, logits reaching about +-20: there an operand rounded to TF32's 10 mantissa bits
  moves a probability by several fp16 ulps.
A GPU test checks, for each scorer over a grid of head_dim, group size, G * window and chunk size, that the native score
call succeeds exactly where the routing predicate says the kernels take the shape, and otherwise reports
"unsupported shape".

Measured on an H100 80GB HBM3 (700 W power limit), where the file runs in about 40 s, with the same figures under both
precisions: ExpectedAttention, SnapKV, ObservedAttention and CriticalKV at most 1 ulp from the rounded fp64 score, at most
0.2 % of a case's positions at 1 ulp, the worst row bias 0.29 of its bound; NonCausal at most 0.35 of its bar (8 fp16
ulps at head_dim 160). With the scales applied to the operands instead, "tf32" put fp16 SnapKV 5 ulps and fp16
ObservedAttention 3 ulps from fp64 on the peaked cases, and 11-15 % of the positions of some ExpectedAttention, SnapKV
and ObservedAttention cases at 1 ulp. Each bar is asserted as stated above, not at the measured values.
"""
import ast
import math
from pathlib import Path

import pytest
import torch

from kvpress_b200 import wide_head_scores as W
from oracle import press_oracle as O
from tests.conftest import ulp16_diff
from tests.gpu_support import (assert_compress, assert_vs_ref64, ckv_assert_scores, ckv_inputs, ea_inputs, ea_ref64,
                               _forced_head, _forced_tail, _name, _native, nca_inputs, nca_ref, oa_inputs, oa_ref64,
                               snap_inputs, snap_ref64, ulp_at)

gpu = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = [torch.bfloat16, torch.float16]
MODULE = Path(W.__file__)


@pytest.fixture(params=["ieee", "tf32"])
def fp32_precision(request):
    """torch's fp32 matmul precision for one test; the caller's setting is restored afterwards."""
    matmul = torch.backends.cuda.matmul
    saved = matmul.fp32_precision
    request.addfinalizer(lambda: setattr(matmul, "fp32_precision", saved))
    matmul.fp32_precision = request.param
    return request.param


def _call(fn, precision: str, *args, **kwargs):
    """One fallback call; the library must not touch the process-wide matmul precision."""
    out = fn(*args, **kwargs)
    assert torch.backends.cuda.matmul.fp32_precision == precision, f"{fn.__name__} changed fp32_precision"
    return out


def _check_compress(sc, k, v, ratio: float = 0.5):
    """native.scores_compress on the fallback's scores: the canonical selection and exact gathers."""
    n_kept = max(1, O.kept_count(k.shape[2], ratio))
    k_out, v_out, idx = _native().scores_compress(sc, k, v, n_kept, return_indices=True)
    assert_compress(k, v, k_out, v_out, idx, sc, n_kept)


# ---------------------------------------------------------------------------------------------------
# the cases: only the arguments that differ from a scorer's defaults
# ---------------------------------------------------------------------------------------------------
OUTSIDE_DIMS = (32, 80, 96, 160, 256)
BIG_GROUPS = (9, 12, 16)

SNAP_DEFAULTS = dict(B=2, D=96, G=4, w=32, S=1500, k=5, chunk=None, peak=False)
SNAP = [
    *[dict(D=D) for D in OUTSIDE_DIMS],
    # G * window past the 512 resident query rows, at the kernels' head dims
    *[dict(D=D, G=G, w=w, S=2000) for D in (64, 128) for G, w in ((16, 64), (12, 64), (8, 65), (9, 57))],
    dict(w=1),
    dict(G=2, S=33),                                   # S = window + 1: one scored position
    *[dict(D=80, G=3, w=16, S=2000, k=k) for k in (1, 3, 7)],
    *[dict(G=3, w=8, S=S, chunk=64) for S in (63, 64, 65, 200)],   # K slabs: chunk - 1, chunk, chunk + 1, 4 slabs
    dict(B=1, D=128, G=9, w=64, S=4097, peak=True),
    dict(B=1, S=4097, peak=True),
]

EA_DEFAULTS = dict(B=2, D=96, G=3, S=2000, cov=True, vn=True, eps=0.0, n_sink=4, chunk=None, peak=False)
EA = [
    *[dict(D=D, S=2500) for D in OUTSIDE_DIMS],
    *[dict(D=D, G=G) for D in (64, 128) for G in BIG_GROUPS],
    dict(D=128, G=16, cov=False), dict(G=9, cov=False),             # the covariance-free scan stops at 8 heads
    *[dict(vn=vn, eps=eps) for vn, eps in ((False, 0.0), (False, 1e-2), (True, 1e-2))],
    *[dict(S=1000, n_sink=n) for n in (0, 1, 999)],
    # slabs of `chunk` logits and of 4 * chunk value norms: L = S - n_sink on both sides of each
    *[dict(S=4 + L, chunk=32) for L in (31, 32, 33, 127, 128, 129)],
    dict(B=1, D=128, G=9, S=4097, peak=True),
    dict(B=1, G=4, S=4097, peak=True),
]

CKV_DEFAULTS = dict(B=2, D=96, G=3, S=700, hidden=600, n_first=70, chunk=None)
CKV = [
    *[dict(D=D) for D in OUTSIDE_DIMS],
    *[dict(G=G) for G in BIG_GROUPS],
    *[dict(G=2, hidden=h) for h in (64, 1000)],
    *[dict(D=80, G=2, S=900, n_first=n) for n in (0, 1, 300, 900)],
    *[dict(G=2, S=S, n_first=S // 10, chunk=64) for S in (63, 64, 65, 200)],
]

OBS_DEFAULTS = dict(B=1, D=96, G=4, S=900, n_q=700, rows=None, peak=False)
OBS = [
    *[dict(D=D, G=2 if D != 96 else 4) for D in OUTSIDE_DIMS],
    *[dict(D=D, G=G) for D in (64, 128) for G in BIG_GROUPS],
    *[dict(B=2, G=2, S=1000, n_q=n) for n in (1, 7, 999, 1000)],
    dict(B=2, G=2, S=300, n_q=20, rows=1),           # blocks of one query row
    dict(B=2, G=2, S=300, n_q=10, rows=3),           # blocks of 3, 3, 3 and 1 rows
    dict(D=128, G=9, S=4097, n_q=1024, peak=True),
    dict(S=4097, n_q=1024, peak=True),
]

NCA_DEFAULTS = dict(B=1, D=96, G=4, S=900, cs=256, chunks=None, peak=False)
NCA = [
    dict(), dict(D=256, G=2, cs=128), dict(D=128, G=16), dict(D=64, G=2, cs=64), dict(D=128, G=2, cs=100),
    dict(D=64, G=4, cs=512),
    *[dict(D=D, G=2, cs=128) for D in (32, 80, 160)],
    *[dict(D=D, G=G, cs=128) for D in (64, 128) for G in (9, 12)], dict(D=64, G=16, cs=128),
    *[dict(B=2, D=64, G=2, S=300, cs=cs) for cs in (1, 2, 129, 512)],          # 512 > S: one padded chunk
    dict(B=2, D=64, G=2, S=201, cs=100, chunks=1),   # S one past two chunks: the padded chunk alone in its block
    dict(B=2, D=64, G=2, S=401, cs=100, chunks=3),   # blocks of 3 + 2 chunks: the padded one inside the second
    dict(S=2048, peak=True),
]

# scores function -> (routing predicate, cases, defaults, the predicate's arguments of a case)
SCORERS = {
    "snapkv_scores": ("snapkv_on_tensor_cores", SNAP, SNAP_DEFAULTS, lambda c: (c["D"], c["G"], c["w"])),
    "expected_attention_scores": ("expected_attention_on_tensor_cores", EA, EA_DEFAULTS,
                                  lambda c: (c["D"], c["G"], c["cov"])),
    "criticalkv_scores": ("criticalkv_on_tensor_cores", CKV, CKV_DEFAULTS, lambda c: (c["D"],)),
    "observed_attention_scores": ("observed_attention_on_tensor_cores", OBS, OBS_DEFAULTS,
                                  lambda c: (c["D"], c["G"])),
    "non_causal_attention_scores": ("non_causal_attention_on_tensor_cores", NCA, NCA_DEFAULTS,
                                    lambda c: (c["D"], c["G"], c["cs"])),
}


def _ids(cases):
    return [f"{i:02d}-" + ("-".join(f"{k}{v}" for k, v in c.items()) or "default") for i, c in enumerate(cases)]


def _full(defaults: dict, case: dict) -> dict:
    assert set(case) <= set(defaults), set(case) - set(defaults)
    return {**defaults, **case}


# ---------------------------------------------------------------------------------------------------
# CPU: the sweep reaches every scores function and every routing condition
# ---------------------------------------------------------------------------------------------------
def _public_functions(suffix: str) -> dict:
    tree = ast.parse(MODULE.read_text())
    return {n.name: n for n in tree.body
            if isinstance(n, ast.FunctionDef) and n.name.endswith(suffix) and not n.name.startswith("_")}


def _conditions(fn: ast.FunctionDef):
    """The conjuncts of a predicate's `return a and b and ...`, each compiled over the predicate's arguments."""
    returns = [n for n in ast.walk(fn) if isinstance(n, ast.Return)]
    assert len(returns) == 1, fn.name
    expr = returns[0].value
    terms = expr.values if isinstance(expr, ast.BoolOp) and isinstance(expr.op, ast.And) else [expr]
    return [(ast.unparse(t), compile(ast.Expression(body=t), fn.name, "eval")) for t in terms]


def test_sweep_reaches_every_scorer_and_every_routing_condition():
    """Every public *_scores function of wide_head_scores.py has cases; every case is one the presses route to it
    (its predicate is False); and every conjunct of every *_on_tensor_cores predicate is False for at least one case,
    so a new function or a new routing condition cannot go untested unnoticed."""
    assert set(SCORERS) == set(_public_functions("_scores"))
    predicates = _public_functions("_on_tensor_cores")
    assert {p for p, *_ in SCORERS.values()} == set(predicates)
    namespace = vars(W)
    for fn_name, (pred_name, cases, defaults, pred_args) in SCORERS.items():
        fn = predicates[pred_name]
        arg_names = [a.arg for a in fn.args.args]
        pred = getattr(W, pred_name)
        full = [_full(defaults, c) for c in cases]
        for c in full:
            assert not pred(*pred_args(c)), f"{fn_name}: {c} is a tensor-core shape"
        for text, code in _conditions(fn):
            false_for = [c for c in full if not eval(code, namespace, dict(zip(arg_names, pred_args(c))))]
            assert false_for, f"{pred_name}: no case drives `{text}` false"


# ---------------------------------------------------------------------------------------------------
# GPU: the routing predicates agree with what the C ABI accepts
# ---------------------------------------------------------------------------------------------------
PRED_DIMS = (32, 64, 80, 96, 128, 256)
PRED_GROUPS = (1, 3, 8, 9, 16)
SNAP_ROWS = ((1, 511), (1, 512), (1, 513), (7, 73), (8, 64), (9, 57), (16, 32), (3, 171), (8, 65))


def _accepts(call) -> bool:
    try:
        call()
    except RuntimeError as e:
        assert "unsupported shape" in str(e), e
        return False
    torch.cuda.synchronize()
    return True


def _shapes(scorer: str):
    """(predicate arguments, native score call) over the grid of one scorer."""
    nat = _native()
    B, H, S, dt = 1, 2, 600, torch.bfloat16
    g = torch.Generator(device=DEV).manual_seed(5)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV).to(dt)  # noqa: E731
    if scorer == "snapkv_scores":
        grid = [(D, G, w) for D in PRED_DIMS for G in PRED_GROUPS for w in (16, 64)]
        grid += [(D, G, w) for D in (64, 96, 128) for G, w in SNAP_ROWS]
        for D, G, w in grid:
            k, q = rn(B, H, S, D), rn(B, H * G, w, D)
            yield (D, G, w), lambda k=k, q=q, w=w: nat.snapkv_score(k, q, w, 5)
    elif scorer == "expected_attention_scores":
        for D in PRED_DIMS:
            for G in PRED_GROUPS:
                k, v, mu = rn(B, H, S, D), rn(B, H, S, D), rn(B, H * G, D)
                cov = rn(B, H * G, D, D) / D
                for c in (cov, None):
                    yield (D, G, c is not None), lambda k=k, v=v, mu=mu, c=c: nat.expected_attention_score(
                        k, v, mu, c, 0.0, 4, True)
    elif scorer == "criticalkv_scores":
        for D in PRED_DIMS:
            for G in PRED_GROUPS:
                v, wo, base = rn(B, H, S, D), rn(256, H * G * D), rn(B, H, S).abs()
                yield (D,), lambda v=v, wo=wo, base=base: nat.criticalkv_score(base, v, wo, 1e-4, 10)
    elif scorer == "observed_attention_scores":
        for D in PRED_DIMS:
            for G in PRED_GROUPS:
                k, q = rn(B, H, S, D), rn(B, H * G, 64, D)
                yield (D, G), lambda k=k, q=q, D=D: nat.observed_attention_score(k, q, D ** -0.5)
    else:
        for D in PRED_DIMS:
            for G in PRED_GROUPS:
                k, v, q = rn(B, H, S, D), rn(B, H, S, D), rn(B, H * G, S, D)
                for cs in (64, 100, 128, 256, 512):
                    yield (D, G, cs), lambda k=k, v=v, q=q, cs=cs: nat.non_causal_attention_score(k, v, q, cs)


@gpu
@pytest.mark.parametrize("scorer", list(SCORERS))
def test_routing_predicate_matches_the_c_abi(scorer, fp32_precision):
    """The native score call succeeds exactly where the press-side predicate sends a shape to the kernels; elsewhere
    it fails with "unsupported shape", so a press never routes a shape to a kernel that refuses it, nor scores a shape
    with GEMMs that a kernel would take."""
    pred = getattr(W, SCORERS[scorer][0])
    wrong = [args for args, call in _shapes(scorer) if _accepts(call) != pred(*args)]
    assert not wrong, f"{scorer}: predicate and C ABI disagree at {wrong}"


# ---------------------------------------------------------------------------------------------------
# GPU: the scorers
# ---------------------------------------------------------------------------------------------------
def _assert_peaked(logits: torch.Tensor, what: str):
    top = float(logits.abs().max())
    assert 15 <= top <= 40, f"{what}: largest |logit| {top:.1f}, meant to be about 20"


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_name)
@pytest.mark.parametrize("case", SNAP, ids=_ids(SNAP))
def test_snapkv_fallback(case, dtype, fp32_precision):
    c = _full(SNAP_DEFAULTS, case)
    B, D, G, w, S, ksz = c["B"], c["D"], c["G"], c["w"], c["S"], c["k"]
    what = f"snapkv {_name(dtype)} {fp32_precision} {case}"
    k, v, q = snap_inputs(B, 2, G, S, D, w, dtype, 3000 + SNAP.index(case))
    if c["peak"]:
        q = (q.float() * 4).to(dtype)  # logits of standard deviation 6
        _assert_peaked(q.double().reshape(B, 2, G * w, D) @ k.double().transpose(-1, -2) / math.sqrt(D), what)
    kw = {} if c["chunk"] is None else {"chunk": c["chunk"]}
    sc = _call(W.snapkv_scores, fp32_precision, k, q, w, ksz, **kw)
    assert_vs_ref64(sc, snap_ref64(q, k, w, ksz), _forced_tail(S, w), what)
    _check_compress(sc, k, v)


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_name)
@pytest.mark.parametrize("case", EA, ids=_ids(EA))
def test_expected_attention_fallback(case, dtype, fp32_precision):
    c = _full(EA_DEFAULTS, case)
    B, D, G, S, n_sink = c["B"], c["D"], c["G"], c["S"], c["n_sink"]
    what = f"ea {_name(dtype)} {fp32_precision} {case}"
    k, v, mu, cov = ea_inputs(B, 2, G, S, D, dtype, 4000 + EA.index(case), cov=c["cov"],
                                 mu_scale=6.0 if c["peak"] else 0.5)
    if c["peak"]:
        _assert_peaked(mu.double().reshape(B, 2, G, D) @ k.double().transpose(-1, -2) / math.sqrt(D), what)
    kw = {} if c["chunk"] is None else {"chunk": c["chunk"]}
    sc = _call(W.expected_attention_scores, fp32_precision, k, v, mu, cov, c["eps"], n_sink, c["vn"], **kw)
    ref = ea_ref64(k, v, mu, cov, c["eps"], n_sink, c["vn"])
    assert_vs_ref64(sc, ref, _forced_head(S, n_sink), what)
    _check_compress(sc, k, v, 0.3)


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_name)
@pytest.mark.parametrize("case", CKV, ids=_ids(CKV))
def test_criticalkv_fallback(case, dtype, fp32_precision):
    c = _full(CKV_DEFAULTS, case)
    B, D, G, S, n_first = c["B"], c["D"], c["G"], c["S"], c["n_first"]
    what = f"ckv {_name(dtype)} {fp32_precision} {case}"
    v, wo, base = ckv_inputs(B, 2, G, S, D, c["hidden"], dtype, seed=5000 + CKV.index(case))
    kw = {} if c["chunk"] is None else {"chunk": c["chunk"]}
    sc = _call(W.criticalkv_scores, fp32_precision, base, v, wo, 1e-4, n_first, **kw)
    ckv_assert_scores(sc, base, v, wo, 1e-4, n_first, what)
    _check_compress(sc, torch.randn_like(v), v)


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_name)
@pytest.mark.parametrize("case", OBS, ids=_ids(OBS))
def test_observed_attention_fallback(case, dtype, fp32_precision):
    c = _full(OBS_DEFAULTS, case)
    B, D, G, S, n_q = c["B"], c["D"], c["G"], c["S"], c["n_q"]
    what = f"obs {_name(dtype)} {fp32_precision} {case}"
    k, v, q = oa_inputs(B, 2, G, S, n_q, D, dtype, seed=6000 + OBS.index(case), q_scale=6.0 if c["peak"] else 1.5)
    if c["peak"]:
        _assert_peaked(q.double().reshape(B, 2, G * n_q, D) @ k.double().transpose(-1, -2) / math.sqrt(D), what)
    max_logits = 1 << 20 if c["rows"] is None else c["rows"] * B * 2 * G * S   # several query blocks either way
    sc = _call(W.observed_attention_scores, fp32_precision, k, q, D ** -0.5, max_logits=max_logits)
    assert_vs_ref64(sc, oa_ref64(k, q, D ** -0.5), torch.zeros(S, dtype=torch.bool), what)
    _check_compress(sc, k, v)


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_name)
@pytest.mark.parametrize("case", NCA, ids=_ids(NCA))
def test_non_causal_attention_fallback(case, dtype, fp32_precision):
    """nca_inputs gives every case logits of standard deviation 6 (chunk maxima of 20-25): all of them are peaked."""
    c = _full(NCA_DEFAULTS, case)
    B, D, G, S, cs = c["B"], c["D"], c["G"], c["S"], c["cs"]
    what = f"nca {_name(dtype)} {fp32_precision} {case}"
    k, v, q = nca_inputs(B, 2, G, S, D, dtype, seed=7000 + NCA.index(case))
    if c["peak"]:
        _assert_peaked(q[..., :cs, :].double().reshape(B, 2, G * cs, D) @ k[..., :cs, :].double().transpose(-1, -2),
                       what)
    max_logits = 1 << 20 if c["chunks"] is None else c["chunks"] * B * 2 * G * cs * cs
    sc = _call(W.non_causal_attention_scores, fp32_precision, k, v, q, cs, max_logits=max_logits)
    z64, E = nca_ref(k, v, q, cs)
    bar = ulp_at(z64, dtype) + 4 * E
    d = (sc.double() - z64).abs()
    assert (d <= bar).all(), f"{what}: {int((d > bar).sum())} positions beyond ulp + 4 E_s ({float((d / bar).max()):.2f})"
    print(f"[measured] {what}: max ulp {int(ulp16_diff(sc, z64.to(dtype)).max())}, "
          f"worst |z - z64| {float((d / bar).max()):.3f} of the bar")
    _check_compress(sc, k, v)
