"""LagKV on the GPU-less box: the C ABI's checks of the two new entry points, the workspace and launch count of the new
scorer id, the argument lists of their wrappers, the float64 definition against the UNMODIFIED reference, and the
press's float32 fallback for lag sizes above the kernel's.

Statuses: every argument of kvp_lagkv_score / kvp_lagkv_compress made invalid on its own (or set to another valid
value), and every pair of such changes to two different arguments, against a restatement of the documented check order
(include/kvpress_b200.h). The pointers are fake, 16-byte aligned or not, and never dereferenced: the calls run in a child
process that sees no GPU, so a call that passes every check fails at its first CUDA call with KVP_ERR_CUDA (-6).

Reference: what the reference's `LagKVPress.score` and `_get_states_score` return on seeded float64 K / V (no bf16
chain and no ties, so the reference computes the definition itself) is stored in tests/golden/lagkv_reference.npz.
To re-record it from a checkout of the reference (located as in oracle/build_ref.py):
    KVP_RECORD_LAGKV=1 python -m pytest tests/test_lagkv_host.py
"""
import ctypes
from pathlib import Path

import pytest
import torch

from kvpress_b200 import LagKVPress, native
from kvpress_b200.presses.lagkv_press import _lagkv_scores_fp32
from tests import abi_cases, lagkv_backend as LB
from tests.abi_cases import GOOD, ODD16
from tests.support import kv, rec, reference_store  # noqa: F401  (rec: fixture)

STORE = Path(__file__).resolve().parent / "golden" / "lagkv_reference.npz"
LAG_MAX = 1024

# --------------------------------------------------------------------------------------------------
# C ABI statuses
# --------------------------------------------------------------------------------------------------
def _checks(f, a, compress):
    """n_sink >= 0 and lag_size >= 1 -> lag_size <= 1024."""
    if a["n_sink"] < 0 or a["L"] < 1:
        return -7
    return -2 if a["L"] > LAG_MAX else 0


ABI = abi_cases.Spec(
    scorer=native.SCORER_LAGKV, fields=dict(Hq=2),
    slots={"kvp_lagkv_score": "K V n_sink L cross scores ws ws_bytes stream",
           "kvp_lagkv_compress": "K V n_sink L cross K_out V_out idx scores ws ws_bytes stream"},
    valid=dict(K=GOOD, V=GOOD, n_sink=4, L=128, cross=0, K_out=GOOD, V_out=GOOD, idx=GOOD, scores=GOOD, ws=GOOD,
               ws_bytes="enough", stream=0),
    changes={
        "p": {"null": None},
        "dtype": {"1": 1, "3": 3},
        "S": {"0": 0, "1": 1},
        "D": {"8": 8, "12": 12, "64": 64, "264": 264},
        "Hq": {"5": 5, "8": 8},
        "n_kept": {"-1": -1, "0": 0, "1000": 1000, "1001": 1001},
        "v_stride": {"s100": (256000, 128000, 100)},
        "K": {"null": None, "odd": ODD16},
        "V": {"null": None, "odd": ODD16},
        "n_sink": {"-1": -1, "0": 0, "1000": 1000, "max": 2 ** 31 - 1},
        "L": {"0": 0, "-3": -3, "1": 1, str(LAG_MAX): LAG_MAX, str(LAG_MAX + 1): LAG_MAX + 1},
        "cross": {"1": 1, "7": 7},
        "K_out": {"null": None, "odd": ODD16},
        "V_out": {"null": None},
        "idx": {"null": None},
        "scores": {"null": None, "odd": ODD16},
        "ws": {"null": None, "odd": ODD16},
        "ws_bytes": {"short": "short"},
    },
    operands={"score": (["K", "V", "scores"], ["K", "V"]), "compress": ([], [])},
    checks=_checks)


def test_every_status_of_the_lagkv_entry_points_follows_the_check_order():
    abi_cases.assert_statuses(__name__, 1400)


def test_workspace_and_launch_count_of_the_new_scorer_id():
    """LagKV needs no scratch of its own: its workspace is the selection stage's. A compress is 3 launches."""
    lib = native.load()
    assert native.SCORER_LAGKV == 9 and native.LAG_MAX == LAG_MAX
    p = native.KvpProblem()
    p.B, p.Hkv, p.Hq, p.D, p.n_kept, p.dtype = 1, 8, 8, 128, 0, 0
    for S in (1, 2, 255, 256, 257, 4096, 131072):
        p.S = S
        lag, generic, n = ctypes.c_size_t(0), ctypes.c_size_t(0), ctypes.c_int(0)
        assert lib.kvp_workspace_bytes(ctypes.byref(p), native.SCORER_LAGKV, ctypes.byref(lag)) == 0
        assert lib.kvp_workspace_bytes(ctypes.byref(p), native.SCORER_GENERIC, ctypes.byref(generic)) == 0
        assert lag.value == generic.value > 0
        assert lib.kvp_launches_per_compress(ctypes.byref(p), native.SCORER_LAGKV, ctypes.byref(n)) == 0
        assert n.value == 3
    assert lib.kvp_launches_per_compress(ctypes.byref(p), 10, ctypes.byref(n)) == -7


# --------------------------------------------------------------------------------------------------
# wrappers: each argument after the kvp_problem, in order, down to the workspace and the stream
# --------------------------------------------------------------------------------------------------
def test_lagkv_wrappers_pass_their_full_argument_list(rec):  # noqa: F811
    P = lambda t: t.data_ptr()  # noqa: E731
    k, v = kv(B=2, H=2, S=300, D=64)

    def last(name, n_kept):
        got, p, a = rec.calls[-1]
        assert got == name and (p["n_kept"], p["Hq"], p["Hkv"], p["D"], p["S"]) == (n_kept, 2, 2, 64, 300)
        problem = native.make_problem(k, v, n_kept)
        assert a[-2:] == [native.workspace_bytes(problem, native.SCORER_LAGKV), 0] and a[-3] != 0
        return a[:-3]

    sc = native.lagkv_score(k, v, 4, 128, False)
    assert last("kvp_lagkv_score", 0) == [P(k), P(v), 4, 128, 0, P(sc)]
    assert sc.shape == (2, 2, 300) and sc.dtype == k.dtype
    native.lagkv_score(k, v, 0, 7, True)
    assert last("kvp_lagkv_score", 0)[2:5] == [0, 7, 1]
    k_out, v_out, idx, sc = native.lagkv_compress(k, v, 16, 32, True, 100, return_indices=True, return_scores=True)
    assert last("kvp_lagkv_compress", 100) == [P(k), P(v), 16, 32, 1, P(k_out), P(v_out), P(idx), P(sc)]
    assert k_out.shape == (2, 2, 100, 64) and idx.dtype == torch.int32
    k_out, v_out, idx, sc = native.lagkv_compress(k, v, 4, 128, False, 100)
    assert idx is None and sc is None
    assert last("kvp_lagkv_compress", 100) == [P(k), P(v), 4, 128, 0, P(k_out), P(v_out), 0, 0]
    # a [..., 8:-4, :] slice of the cache goes to the library in place, with its own strides (ChunkPress)
    ks, vs = k[:, :, 8:-4], v[:, :, 8:-4]
    native.lagkv_score(ks, vs, 4, 16, False)
    got, p, a = rec.calls[-1]
    assert a[:2] == [P(ks), P(vs)] and p["S"] == 288 and p["k_stride"] == (2 * 300 * 64, 300 * 64, 64)
    # n_kept == 0: nothing is enqueued
    n = len(rec.calls)
    native.lagkv_compress(k, v, 4, 128, False, 0)
    assert len(rec.calls) == n


# --------------------------------------------------------------------------------------------------
# the float64 definition against the unmodified reference
# --------------------------------------------------------------------------------------------------
ref = reference_store(STORE, "KVP_RECORD_LAGKV")


# (name, S, n_sink, lag_size, planted constant channel)
DEFINITION = [
    ("short", 35, 4, 16, False),           # S = n_sink + 2L - 1
    ("two", 36, 4, 16, False),             # S = n_sink + 2L: one scored partition
    ("three-1", 51, 4, 16, False),         # n_sink + 3L - 1: one scored partition, a tail of 2L - 1
    ("several", 105, 4, 16, False),        # six partitions and a remainder of 5
    ("no-sink", 70, 0, 16, False),
    ("sink-eq-s", 40, 40, 16, False),
    ("sink-gt-s", 40, 50, 16, False),
    ("lag1", 10, 4, 1, False),             # every reference partition is one row: NaN
    ("lag7", 42, 4, 7, False),
    ("lag100", 321, 4, 100, False),
    ("lag128", 397, 4, 128, False),
    ("constant", 105, 4, 16, True),        # a constant K channel in partition 3, a constant V channel in partition 5
]


def _definition_inputs(S, n_sink, L, planted):
    g = torch.Generator().manual_seed(S * 31 + n_sink * 7 + L)
    k = torch.randn(1, 2, S, 16, generator=g, dtype=torch.float64) * 1.5
    v = torch.randn(1, 2, S, 16, generator=g, dtype=torch.float64)
    if planted:
        k[:, 0, n_sink + 3 * L:n_sink + 4 * L, 5] = 0.25
        v[:, 1, n_sink + 5 * L:n_sink + 6 * L, 2] = -1.0
    return k, v


@pytest.mark.parametrize("cross", [False, True], ids=["rank", "cross"])
@pytest.mark.parametrize("name,S,n_sink,L,planted", DEFINITION, ids=[d[0] for d in DEFINITION])
def test_float64_definition_is_the_reference(ref, name, S, n_sink, L, planted, cross):
    """The float64 definition of tests/lagkv_backend.py against the reference's own score() and _get_states_score on
    float64 inputs: ranks exactly, cross scores and the states to 1e-12 relative, NaN where the reference has NaN."""
    k, v = _definition_inputs(S, n_sink, L, planted)

    def reference(kvpress):
        press = kvpress.presses.lagkv_press.LagKVPress(compression_ratio=0.5, n_sink=n_sink, lag_size=L,
                                                       cross_scoring=cross)
        out = {"score": press.score(None, None, k, v, None, None)}
        if not LB.is_short(S, n_sink, L):
            P = (S - n_sink) // L
            out["states_k"] = press._get_states_score(k[:, :, n_sink:n_sink + P * L].view(1, 2, P, L, 16))
        return out

    want = ref(f"definition/{name}/{int(cross)}", reference)
    got = LB.lagkv_scores64(k, v, n_sink, L, cross)
    score = torch.as_tensor(want["score"], dtype=torch.float64)
    assert got.shape == score.shape == (1, 2, S)
    assert torch.equal(torch.isnan(got), torch.isnan(score))
    if cross:
        assert torch.allclose(got.nan_to_num(), score.nan_to_num(), rtol=1e-12, atol=0)
    else:
        assert torch.equal(got, score)  # the ranks, exactly
    if "states_k" in want:
        states = torch.as_tensor(want["states_k"], dtype=torch.float64)
        mine = LB.sigma64(k, n_sink, L).softmax(dim=-1)
        assert torch.equal(torch.isnan(mine), torch.isnan(states))
        assert torch.allclose(mine.nan_to_num(), states.nan_to_num(), rtol=1e-12, atol=0)
    if planted:  # the partitions referenced by a constant channel are NaN in the reference too
        assert torch.isnan(score[0, 0, n_sink + 2 * L:n_sink + 3 * L]).all() == cross
        assert torch.isnan(score[0, 1, n_sink + 4 * L:n_sink + 5 * L]).all() == cross
        if not cross:  # NaN partitions rank in position order
            assert torch.equal(score[0, 0, n_sink + 2 * L:n_sink + 3 * L],
                               (torch.arange(L, dtype=torch.float32) / L).double())


@pytest.mark.parametrize("cross", [False, True], ids=["rank", "cross"])
@pytest.mark.parametrize("name,S,n_sink,L,planted", DEFINITION, ids=[d[0] for d in DEFINITION])
def test_float32_fallback_follows_the_definition(name, S, n_sink, L, planted, cross):
    """The press's torch float32 evaluation (lag_size above the kernel's) against the float64 definition, both rounded
    to bf16: the sinks, tail and ramp exactly, ranks equal, cross scores within one bf16 ulp."""
    k, v = _definition_inputs(S, n_sink, L, planted)
    kb, vb = k.to(torch.bfloat16), v.to(torch.bfloat16)
    got = _lagkv_scores_fp32(kb, vb, n_sink, L, cross)
    want = LB.lagkv_score(kb, vb, n_sink, L, cross)
    assert got.dtype == torch.bfloat16 and torch.equal(torch.isnan(got), torch.isnan(want))
    if cross:
        d = (got.float() - want.float()).abs().nan_to_num()
        assert (d <= want.float().abs().nan_to_num() * 2 ** -7).all()
    else:
        assert torch.equal(got, want)


def test_press_mirrors_the_reference_fields():
    press = LagKVPress()
    assert (press.compression_ratio, press.n_sink, press.lag_size, press.cross_scoring) == (0.0, 4, 128, False)
    assert LagKVPress.needs_hidden_states is False
