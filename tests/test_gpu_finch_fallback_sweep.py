"""FinchPress's torch GEMM score fallback (kvpress_b200/finch_wide_head.py) against float64, at every kind of shape the
press routes to it, under both of torch's fp32 matmul precisions; and the press's selection on those scores.

`finch_scores` scores the shapes `kvp_finch_*` does not instantiate (head_dim other than 64 / 128, more than 8 query
heads per kv head) with fp32 GEMMs in blocks of window rows, under the contract of the kernels: fp32 evaluation of the
formula, rounded once to the cache dtype. As in tests/test_gpu_wide_head_sweep.py, every GPU case runs under
torch.backends.cuda.matmul.fp32_precision = "ieee" and "tf32": every GEMM operand is an exact 16-bit value and the
1/sqrt(D) scale multiplies the fp32 products, so TF32 rounds nothing, both precisions meet the same bar, and the call
leaves the setting as it found it.

Bar: that of tests/test_gpu_finch.py (`gpu_support.assert_scores`): every context score within 1 ulp of the float64
value, the window holding round(max + 1); and, where a row has at least BIAS_MIN_N context positions, the row-bias bar of
`gpu_support.assert_vs_ref64`.

Cases: head_dim 32 / 80 / 96 / 160 / 256; head_dim 64 / 128 with 9, 12 and 16 query heads per kv head; bf16 and fp16;
normalize on and off; window 1 and S - 1; B = 2 (the block of window rows depends on B); a small `max_logits`, so the
block is 1, w - 1, w and w + 1 window rows; one peaked case with logits near +-20, where a scale applied to the
operands moves TF32-rounded fp16 probabilities by several ulps. A GPU test checks over a grid of head_dim x group size
that `native.finch_score` succeeds exactly where `finch_on_tensor_cores` sends a shape to the kernels, and otherwise
reports "unsupported shape"; a CPU test that every public function and every routing condition is reached. The press
test runs `FinchPress.compress` on fallback shapes, chunked and not, with and without key re-rotation: its rows are the
chunked canonical selection (`gpu_support.chunked_canonical`) of `finch_scores` with the window set to +inf.

Measured on an H100 80GB HBM3 (700 W power limit): every case passes under both precisions, and no case found a bug in
the module. With the scale applied to the operands instead, "tf32" put the peaked fp16 cases 5-7 ulps from the float64
scores and the peaked bf16 case just past 1 ulp, while "ieee" still passed. Each bar is asserted as stated above, not at
the measured values.
"""
import ast
import math
from pathlib import Path
from types import SimpleNamespace

import pytest
import torch

from kvpress_b200 import FinchPress, finch_wide_head as F
from tests.gpu_support import (BIAS_MIN_N, _bits, _forced_tail, _gather, _name, _native, assert_gather, assert_idx,
                               assert_scores, assert_vs_ref64, chunked_canonical, rerotation_admissible, rope_inv_freq,
                               scores64)

gpu = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = [torch.bfloat16, torch.float16]
MODULE = Path(F.__file__)


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


def inputs(B, H, G, S, D, w, dtype, seed, q_scale=1.5):
    g = torch.Generator(device=DEV).manual_seed(seed)
    k = torch.randn(B, H, S, D, generator=g, device=DEV).to(dtype)
    q = (torch.randn(B, H * G, w, D, generator=g, device=DEV) * q_scale).to(dtype)
    v = torch.randn(B, H, S, D, generator=g, device=DEV).to(dtype)
    return k, v, q


# ---------------------------------------------------------------------------------------------------
# the cases: only the arguments that differ from the defaults
# ---------------------------------------------------------------------------------------------------
OUTSIDE_DIMS = (32, 80, 96, 160, 256)
BIG_GROUPS = (9, 12, 16)
DEFAULTS = dict(B=1, D=96, G=4, S=700, w=33, normalize=True, rows=None, peak=False)
CASES = [
    *[dict(D=D) for D in OUTSIDE_DIMS],
    *[dict(D=D, G=G) for D in (64, 128) for G in BIG_GROUPS],
    dict(normalize=False), dict(D=160, G=9, normalize=False),
    dict(w=1), dict(w=699), dict(S=40, w=39, G=2),
    dict(B=2, S=900), dict(B=2, D=128, G=12, S=900, w=60),
    *[dict(B=2, G=2, S=300, w=12, rows=r) for r in (1, 11, 12, 13)],   # blocks of window rows: 1, w - 1, w, w + 1
    dict(S=2048, w=64, peak=True),
    dict(D=128, G=9, S=2048, w=64, peak=True),
]


def _full(case: dict) -> dict:
    assert set(case) <= set(DEFAULTS), set(case) - set(DEFAULTS)
    return {**DEFAULTS, **case}


def _ids(cases):
    return [f"{i:02d}-" + ("-".join(f"{k}{v}" for k, v in c.items()) or "default") for i, c in enumerate(cases)]


# ---------------------------------------------------------------------------------------------------
# CPU: every public function and every routing condition is reached
# ---------------------------------------------------------------------------------------------------
def test_sweep_reaches_every_function_and_every_routing_condition():
    """finch_wide_head.py has one scores function and one routing predicate; every case is one the press routes to
    the fallback, and every conjunct of the predicate is False for at least one case."""
    tree = ast.parse(MODULE.read_text())
    public = {n.name: n for n in tree.body if isinstance(n, ast.FunctionDef) and not n.name.startswith("_")}
    assert set(public) == {"finch_scores", "finch_on_tensor_cores"}
    pred = public["finch_on_tensor_cores"]
    returns = [n for n in ast.walk(pred) if isinstance(n, ast.Return)]
    assert len(returns) == 1
    expr = returns[0].value
    terms = expr.values if isinstance(expr, ast.BoolOp) and isinstance(expr.op, ast.And) else [expr]
    full = [_full(c) for c in CASES]
    for c in full:
        assert not F.finch_on_tensor_cores(c["D"], c["G"]), f"{c} is a tensor-core shape"
    arg_names = [a.arg for a in pred.args.args]
    for t in terms:
        code = compile(ast.Expression(body=t), pred.name, "eval")
        false_for = [c for c in full if not eval(code, vars(F), dict(zip(arg_names, (c["D"], c["G"]))))]
        assert false_for, f"no case drives `{ast.unparse(t)}` false"
    # the press routes with this predicate
    assert "finch_wide_head.finch_on_tensor_cores(" in (MODULE.parent / "presses" / "finch_press.py").read_text()


# ---------------------------------------------------------------------------------------------------
# GPU: the routing predicate agrees with what the C ABI accepts
# ---------------------------------------------------------------------------------------------------
PRED_DIMS = (32, 64, 80, 96, 128, 256)
PRED_GROUPS = (1, 3, 8, 9, 16)


@gpu
def test_routing_predicate_matches_the_c_abi(fp32_precision):
    nat = _native()
    g = torch.Generator(device=DEV).manual_seed(5)
    wrong = []
    for D in PRED_DIMS:
        for G in PRED_GROUPS:
            k = torch.randn(1, 2, 600, D, generator=g, device=DEV).to(torch.bfloat16)
            q = torch.randn(1, 2 * G, 16, D, generator=g, device=DEV).to(torch.bfloat16)
            try:
                nat.finch_score(k, q, 16)
                torch.cuda.synchronize()
                accepted = True
            except RuntimeError as e:
                assert "unsupported shape" in str(e), e
                accepted = False
            if accepted != F.finch_on_tensor_cores(D, G):
                wrong.append((D, G))
    assert not wrong, f"predicate and C ABI disagree at {wrong}"
    assert torch.backends.cuda.matmul.fp32_precision == fp32_precision


# ---------------------------------------------------------------------------------------------------
# GPU: the scores
# ---------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_name)
@pytest.mark.parametrize("case", CASES, ids=_ids(CASES))
def test_finch_fallback(case, dtype, fp32_precision):
    c = _full(case)
    B, D, G, S, w = c["B"], c["D"], c["G"], c["S"], c["w"]
    what = f"finch {_name(dtype)} {fp32_precision} {case}"
    k, _, q = inputs(B, 2, G, S, D, w, dtype, 8000 + CASES.index(case), q_scale=6.0 if c["peak"] else 1.5)
    if c["peak"]:  # logits of standard deviation 6
        top = float((q.double().reshape(B, 2, G * w, D) @ k.double().transpose(-1, -2)).abs().max()) / math.sqrt(D)
        assert 15 <= top <= 40, f"{what}: largest |logit| {top:.1f}, meant to be about 20"
    kw = {} if c["rows"] is None else {"max_logits": c["rows"] * B * 2 * G * S}
    sc = _call(F.finch_scores, fp32_precision, k, q, w, c["normalize"], **kw)
    assert sc.dtype == dtype and sc.shape == (B, 2, S)
    assert_scores(sc, k, q, w, c["normalize"], what)
    if S - w >= BIAS_MIN_N:
        ref = torch.nn.functional.pad(scores64(k, q, w, c["normalize"]), (0, w), value=math.inf)
        assert_vs_ref64(sc, ref, _forced_tail(S, w), what)


# ---------------------------------------------------------------------------------------------------
# GPU: the press on fallback shapes
# ---------------------------------------------------------------------------------------------------
PRESS = [(D, G, L, rerotate) for D, G in ((96, 4), (64, 12)) for L in (None, 700) for rerotate in (False, True)]


@gpu
@pytest.mark.parametrize("D,G,L,rerotate", PRESS, ids=[f"d{D}-g{G}-L{L}-rerot{int(r)}" for D, G, L, r in PRESS])
def test_press_on_fallback_shapes(D, G, L, rerotate, fp32_precision):
    """FinchPress.compress: cuBLAS scores, then the sm_90a selection with the window forced; the kept rows are the
    chunked canonical selection of finch_scores with the window at +inf (unchunked: one chunk of the whole row)"""
    S, w, r = 2101, 30, 0.5
    dtype = torch.float16 if G == 12 else torch.bfloat16
    k, v, q = inputs(1, 2, G, S, D, w, dtype, seed=D + G)
    inv = rope_inv_freq("theta10000", D)
    press = FinchPress(r, chunk_length=L, rerotate_keys=rerotate)
    press.window_size = w
    press.window_queries = lambda *a: q
    module = SimpleNamespace(rotary_emb=SimpleNamespace(inv_freq=inv))
    k_out, v_out = _call(press.compress, fp32_precision, module, None, k, v, None, {})
    scores = F.finch_scores(k, q, w, True)
    scores[..., -w:] = float("inf")
    _, ck, tk, n = _native().chunk_counts(S, L, r)
    want = chunked_canonical(scores, L, ck, tk) if L else chunked_canonical(scores, S, n, 0)
    assert k_out.shape[2] == want.shape[-1]
    assert_gather(v_out, v, want, "V'")
    if rerotate:
        adm = _bits(rerotation_admissible(k, want, inv))
        assert (adm == _bits(k_out)[None]).any(0).all(), "K' not an admissible re-rotation"
    else:
        assert_gather(k_out, k, want, "K'")
    # the kept positions are those of the entry points' own idx
    idx = _native().scores_compress_chunked(scores, k, v, r, L, None, True)[2] if L else \
        _native().scores_compress(scores, k, v, n, return_indices=True)[2]
    assert_idx(idx, want, "idx")
    assert torch.equal(_bits(_gather(v, idx)), _bits(v_out))
