"""CUR on the GPU-less box: the C ABI's checks of the two new entry points, the workspace and launch count of the new
scorer id, the argument lists of their wrappers, the float64 definition against the UNMODIFIED reference, the press's
float32 fallback for windows above the kernel's, and the press alone and under the wrapper presses on tiny Llamas with
the float64 stand-ins of tests/cur_backend.py in place of the kernels.

Statuses: every argument of kvp_cur_score / kvp_cur_compress made invalid on its own (or set to another valid value),
and every pair of such changes to two different arguments, against a restatement of the documented check order
(include/kvpress_b200.h). The pointers are fake, 16-byte aligned or not, and never dereferenced: the calls run in a child
process that sees no GPU, so a call that passes every check fails at its first CUDA call with KVP_ERR_CUDA (-6).

Reference: what the reference's `CURPress.score` returns on seeded float32 K / V, and the rows its press keeps on
float32 tiny Llamas, are stored in tests/golden/cur_reference.npz. To re-record it from a checkout of the reference
(located as in oracle/build_ref.py):
    KVP_RECORD_CUR=1 python -m pytest tests/test_cur_host.py
"""
import ctypes
import itertools
import math
from pathlib import Path

import pytest
import torch
from transformers import DynamicCache

from kvpress_b200 import (AdaKVPress, ChunkPress, ComposedPress, CriticalKVPress, CURPress, DecodingPress,
                          KeyRerotationPress, KnormPress, native)
from kvpress_b200.presses.cur_press import _cur_scores_fp32
from oracle import press_oracle as O
from tests import abi_cases, cpu_backend, criticalkv_backend, cur_backend as CB
from tests.abi_cases import GOOD, ODD16
from tests.support import close, kv, rec, reference_store, rows_signature  # noqa: F401  (rec: fixture)
from tests.tiny_models import distinct_ids, tiny_model

STORE = Path(__file__).resolve().parent / "golden" / "cur_reference.npz"
WINDOW_MAX, RANK_MAX = 1024, 32
TYPES = CB.LEVERAGE_TYPES

# --------------------------------------------------------------------------------------------------
# C ABI statuses
# --------------------------------------------------------------------------------------------------
def _checks(f, a, compress):
    """num_sinks, leverage_type, local_window_size, r and G / r together -> the kernel's window and r limits."""
    if a["sinks"] < 0 or not 0 <= a["type"] <= 3 or a["w"] < 0 or a["r"] < 0 or (a["G"] is None) != (a["r"] == 0):
        return -7
    return -2 if a["w"] > WINDOW_MAX or a["r"] > RANK_MAX else 0


ABI = abi_cases.Spec(
    scorer=native.SCORER_CUR, fields=dict(Hq=2),
    slots={"kvp_cur_score": "K V sinks type w G r scores ws ws_bytes stream",
           "kvp_cur_compress": "K V sinks type w G r K_out V_out idx scores ws ws_bytes stream"},
    valid=dict(K=GOOD, V=GOOD, sinks=4, type=3, w=16, G=None, r=0, K_out=GOOD, V_out=GOOD, idx=GOOD, scores=GOOD,
               ws=GOOD, ws_bytes="enough", stream=0),
    changes={
        "p": {"null": None},
        "dtype": {"1": 1, "3": 3},
        "S": {"0": 0, "1": 1},
        "D": {"8": 8, "12": 12, "264": 264},
        "Hq": {"5": 5, "8": 8},
        "n_kept": {"-1": -1, "0": 0, "1000": 1000, "1001": 1001},
        "v_stride": {"s100": (256000, 128000, 100)},
        "K": {"null": None, "odd": ODD16},
        "V": {"null": None, "odd": ODD16},
        "sinks": {"-1": -1, "0": 0, "1000": 1000, "max": 2 ** 31 - 1},
        "type": {"-1": -1, "0": 0, "2": 2, "4": 4},
        "w": {"-3": -3, "0": 0, "1": 1, str(WINDOW_MAX): WINDOW_MAX, str(WINDOW_MAX + 1): WINDOW_MAX + 1},
        "G": {"set": GOOD, "odd": ODD16},
        "r": {"-1": -1, "20": 20, str(RANK_MAX): RANK_MAX, str(RANK_MAX + 1): RANK_MAX + 1},
        "K_out": {"null": None, "odd": ODD16},
        "V_out": {"null": None},
        "idx": {"null": None},
        "scores": {"null": None, "odd": ODD16},
        "ws": {"null": None, "odd": ODD16},
        "ws_bytes": {"short": "short"},
    },
    operands={"score": (["K", "V", "scores"], ["K", "V"]), "compress": ([], [])},
    checks=_checks)


def test_every_status_of_the_cur_entry_points_follows_the_check_order():
    want = abi_cases.assert_statuses(__name__, 1900)
    # a projection and its column count are one operand: both given is valid, and the limits are the kernel's
    assert want["kvp_cur_score(G=set,r=20)"] == -6 and want["kvp_cur_score(G=set,r=33)"] == -2
    assert want["kvp_cur_score(G=set)"] == want["kvp_cur_score(r=20)"] == -7


def test_workspace_and_launch_count_of_the_new_scorer_id():
    """CUR's workspace is the selection stage's plus u as fp32 [B Hkv, S] and one fp64 partial per 256 positions, each
    rounded up to 256 bytes. A compress is 4 launches. The id is 11; 10 is not assigned."""
    lib = native.load()
    assert native.SCORER_CUR == 11 and native.SCORER_LAGKV == 9
    assert (native.CUR_WINDOW_MAX, native.CUR_RANK_MAX) == (WINDOW_MAX, RANK_MAX)
    assert native.CUR_LEVERAGE_TYPES == TYPES
    p = native.KvpProblem()
    p.B, p.Hkv, p.Hq, p.D, p.n_kept, p.dtype = 1, 8, 8, 128, 0, 0
    up = lambda x: -(-x // 256) * 256  # noqa: E731
    for S in (1, 2, 255, 256, 257, 4096, 131072):
        p.S = S
        cur, generic, n = ctypes.c_size_t(0), ctypes.c_size_t(0), ctypes.c_int(0)
        assert lib.kvp_workspace_bytes(ctypes.byref(p), native.SCORER_CUR, ctypes.byref(cur)) == 0
        assert lib.kvp_workspace_bytes(ctypes.byref(p), native.SCORER_GENERIC, ctypes.byref(generic)) == 0
        assert cur.value == generic.value + up(8 * S * 4) + up(8 * -(-S // 256) * 8)
        assert lib.kvp_launches_per_compress(ctypes.byref(p), native.SCORER_CUR, ctypes.byref(n)) == 0
        assert n.value == 4
    for unknown in (10, 12):  # 10 stays unassigned
        assert lib.kvp_launches_per_compress(ctypes.byref(p), unknown, ctypes.byref(n)) == -7


# --------------------------------------------------------------------------------------------------
# wrappers: each argument after the kvp_problem, in order, down to the workspace and the stream
# --------------------------------------------------------------------------------------------------
def test_cur_wrappers_pass_their_full_argument_list(rec):  # noqa: F811
    P = lambda t: t.data_ptr()  # noqa: E731
    k, v = kv(B=2, H=2, S=300, D=64)
    G = torch.randn(64, 20)

    def last(name, n_kept):
        got, p, a = rec.calls[-1]
        assert got == name and (p["n_kept"], p["Hq"], p["Hkv"], p["D"], p["S"]) == (n_kept, 2, 2, 64, 300)
        problem = native.make_problem(k, v, n_kept)
        assert a[-2:] == [native.workspace_bytes(problem, native.SCORER_CUR), 0] and a[-3] != 0
        return a[:-3]

    sc = native.cur_score(k, v, 4, "kv_product", 16)
    assert last("kvp_cur_score", 0) == [P(k), P(v), 4, 3, 16, 0, 0, P(sc)]
    assert sc.shape == (2, 2, 300) and sc.dtype == k.dtype
    for i, name in enumerate(TYPES):
        native.cur_score(k, v, 0, name, 0, G)
        assert last("kvp_cur_score", 0)[2:7] == [0, i, 0, P(G), 20]
    k_out, v_out, idx, sc = native.cur_compress(k, v, 16, "key", 32, G, 100, return_indices=True, return_scores=True)
    assert last("kvp_cur_compress", 100) == [P(k), P(v), 16, 0, 32, P(G), 20, P(k_out), P(v_out), P(idx), P(sc)]
    assert k_out.shape == (2, 2, 100, 64) and idx.dtype == torch.int32
    k_out, v_out, idx, sc = native.cur_compress(k, v, 4, "kv_avg", 16, None, 100)
    assert idx is None and sc is None
    assert last("kvp_cur_compress", 100) == [P(k), P(v), 4, 2, 16, 0, 0, P(k_out), P(v_out), 0, 0]
    # a [..., 8:-4, :] slice of the cache goes to the library in place, with its own strides (ChunkPress)
    ks, vs = k[:, :, 8:-4], v[:, :, 8:-4]
    native.cur_score(ks, vs, 4, "kv_product", 16)
    got, p, a = rec.calls[-1]
    assert a[:2] == [P(ks), P(vs)] and p["S"] == 288 and p["k_stride"] == (2 * 300 * 64, 300 * 64, 64)
    # a projection of another dtype, shape or layout
    with pytest.raises(RuntimeError, match="float32 projection"):
        native.cur_score(k, v, 4, "key", 16, G.double())
    with pytest.raises(RuntimeError, match="float32 projection"):
        native.cur_score(k, v, 4, "key", 16, torch.randn(32, 20))
    native.cur_score(k, v, 4, "key", 16, torch.randn(20, 64).t())  # copied to row-major
    assert last("kvp_cur_score", 0)[5] != 0
    with pytest.raises(ValueError, match="Unknown leverage type"):
        native.cur_score(k, v, 4, "kv", 16)
    # n_kept == 0: nothing is enqueued
    n = len(rec.calls)
    native.cur_compress(k, v, 4, "kv_product", 16, None, 0)
    assert len(rec.calls) == n


# --------------------------------------------------------------------------------------------------
# the float64 definition against the unmodified reference
# --------------------------------------------------------------------------------------------------
ref = reference_store(STORE, "KVP_RECORD_CUR")


# (S, local_window_size): S a multiple of w, one more, one less, S below w, w = 1
SHAPES = [(64, 16), (65, 16), (47, 16), (9, 16), (23, 1), (50, 7)]
SINKS = (0, 4, 70)


def _definition_inputs(S, w):
    g = torch.Generator().manual_seed(S * 31 + w)
    k = torch.randn(1, 2, S, 16, generator=g) * 1.5
    v = torch.randn(1, 2, S, 16, generator=g)
    return k, v


def _draw(D: int, seed: int) -> torch.Tensor:
    """The projection the reference and the press draw after torch.manual_seed(seed)."""
    torch.manual_seed(seed)
    return torch.randn(D, 20) / math.sqrt(20)


@pytest.mark.parametrize("projected", [False, True], ids=["plain", "projected"])
@pytest.mark.parametrize("local", [True, False], ids=["local", "global"])
@pytest.mark.parametrize("leverage_type", TYPES)
def test_float64_definition_is_the_reference(ref, leverage_type, local, projected):
    """The float64 definition of tests/cur_backend.py against the reference's own score() on float32 inputs, to float32
    rounding; the sinks exactly."""
    for (S, w), sinks in itertools.product(SHAPES, SINKS):
        k, v = _definition_inputs(S, w)

        def reference(kvpress):
            press = kvpress.presses.cur_press.CURPress(
                compression_ratio=0.5, num_sinks=sinks, leverage_type=leverage_type, use_random_leverage=projected,
                use_local_approximation=local, local_window_size=w)
            torch.manual_seed(S + sinks)
            return {"score": press.score(None, None, k, v, None, None)}

        want = ref(f"definition/{leverage_type}/{int(local)}/{int(projected)}/{S}/{w}/{sinks}", reference)
        score = torch.as_tensor(want["score"], dtype=torch.float64)
        G = _draw(16, S + sinks) if projected else None
        got = CB.cur_scores64(k, v, sinks, leverage_type, w if local else 0, G)
        assert got.shape == score.shape == (1, 2, S)
        assert torch.equal(got[..., :sinks], torch.ones_like(got[..., :sinks]))
        assert torch.allclose(got, score, rtol=2e-5, atol=0), (S, w, sinks, float((got / score - 1).abs().max()))
        if sinks < S:  # the row sum runs over every position, the sinks included
            assert got[..., sinks:].sum(dim=-1).max() <= 1 + 1e-12
            u = CB.combined64(k, v, leverage_type, w if local else 0, G)
            assert torch.allclose(got[..., sinks:], (u / u.sum(dim=-1, keepdim=True))[..., sinks:], rtol=1e-15)


def test_unknown_leverage_type_and_negative_sinks():
    k, v = _definition_inputs(40, 16)
    with pytest.raises(ValueError, match="Unknown leverage type: choose from 'kv_avg', 'key', 'value' or 'kv_product'"):
        CURPress(0.5, leverage_type="kv").score(None, None, k, v, None, {})
    with pytest.raises(ValueError, match="num_sinks"):
        CURPress(0.5, num_sinks=-1).score(None, None, k, v, None, {})
    with pytest.raises(ValueError, match="local_window_size"):
        CURPress(0.5, local_window_size=0).score(None, None, k, v, None, {})


def test_zero_windows_and_nan_inputs_propagate():
    """An all-zero window is 0/0: the row's non-sink scores are all NaN. A zero row inside a non-zero window scores 0.
    A NaN input makes its row NaN. Other rows are untouched. As the reference does."""
    k, v = _definition_inputs(80, 16)
    k[0, 0, 32:48] = 0       # window 2 of row 0 has no key mass
    v[0, 1, 5] = 0           # one zero value row inside a non-zero window
    got = CB.cur_scores64(k, v, 4, "kv_product", 16)
    assert torch.isnan(got[0, 0, 4:]).all() and (got[0, 0, :4] == 1).all()
    assert got[0, 1, 5] == 0 and torch.isfinite(got[0, 1]).all() and (got[0, 1, 6:] > 0).all()
    assert torch.isfinite(CB.cur_scores64(k, v, 4, "value", 16)[0, 0]).all()  # "value" does not read the keys
    assert torch.isfinite(CB.cur_scores64(k, v, 4, "kv_product", 0)).all()    # no windows: no 0/0
    k, v = _definition_inputs(80, 16)
    v[0, 1, 70, 3] = float("nan")
    got = CB.cur_scores64(k, v, 4, "kv_avg", 16)
    assert torch.isnan(got[0, 1, 4:]).all() and torch.isfinite(got[0, 0]).all()
    sc16 = CB.cur_score(k.bfloat16(), v.bfloat16(), 4, "kv_avg", 16)
    assert sc16.dtype == torch.bfloat16 and torch.isnan(sc16[0, 1, 4:]).all()
    # the shared selection ranks NaN above every number, the sinks' 1 included: a NaN row keeps its first non-sink
    # positions, and the sinks only once every NaN position is kept
    idx = O.select_lowest_index_ties(sc16, 10)
    assert idx[0, 1].tolist() == list(range(4, 14))
    assert O.select_lowest_index_ties(sc16, 78)[0, 1].tolist() == [0, 1, *range(4, 80)]


@pytest.mark.parametrize("projected", [False, True], ids=["plain", "projected"])
@pytest.mark.parametrize("leverage_type", TYPES)
def test_float32_fallback_follows_the_definition(leverage_type, projected):
    """The press's torch float32 evaluation (windows above the kernel's) against the float64 definition, both rounded to
    bf16: within one bf16 ulp, the sinks exactly."""
    g = torch.Generator().manual_seed(3)
    k = torch.randn(1, 2, 2600, 16, generator=g).bfloat16()
    v = torch.randn(1, 2, 2600, 16, generator=g).bfloat16()
    G = _draw(16, 9) if projected else None
    for w in (WINDOW_MAX + 1, 3000, 0, 16):
        got = _cur_scores_fp32(k, v, 4, leverage_type, w, G)
        want = CB.cur_score(k, v, 4, leverage_type, w, G)
        assert got.dtype == torch.bfloat16 and (got[..., :4] == 1).all()
        assert ((got.float() - want.float()).abs() <= want.float().abs() * 2 ** -7).all()


def test_press_mirrors_the_reference_fields():
    press = CURPress()
    assert (press.compression_ratio, press.num_sinks, press.leverage_type, press.use_random_leverage,
            press.use_local_approximation, press.local_window_size) == (0.0, 4, "kv_product", False, True, 16)
    assert CURPress.needs_hidden_states is False
    assert CURPress(0.5).compression_ratio == 0.5


def test_press_arguments_and_the_projection_draw(monkeypatch):
    """What the press hands to native.cur_score / cur_compress: window 0 without local approximation, and with
    use_random_leverage the float32 G = randn(D, 20) / sqrt(20) of the global generator, drawn anew on every call."""
    calls = []
    monkeypatch.setattr(native, "cur_score", lambda *a: calls.append(a) or torch.zeros(a[0].shape[:3]))
    monkeypatch.setattr(native, "cur_compress", lambda *a: calls.append(a) or (a[0], a[1], None, None))
    k, v = _definition_inputs(64, 16)
    CURPress(0.5).score(None, None, k, v, None, {})
    assert calls[-1][2:] == (4, "kv_product", 16, None)
    CURPress(0.5, use_local_approximation=False, leverage_type="key", num_sinks=0).score(None, None, k, v, None, {})
    assert calls[-1][2:] == (0, "key", 0, None)
    press = CURPress(0.5, use_random_leverage=True)
    torch.manual_seed(123)
    press.score(None, None, k, v, None, {})
    press.compress(None, None, k, v, None, {})
    torch.manual_seed(123)
    first, second = torch.randn(16, 20) / math.sqrt(20), torch.randn(16, 20) / math.sqrt(20)
    assert calls[-2][5].dtype == torch.float32 and torch.equal(calls[-2][5], first)
    assert torch.equal(calls[-1][5], second) and calls[-1][6] == 32
    # a window above the kernel's: the float32 evaluation and the shared selection
    monkeypatch.setattr(native, "scores_compress", lambda sc, kk, vv, n: calls.append(("generic", n)) or (kk, vv, None))
    n = len(calls)
    big = CURPress(0.5, local_window_size=WINDOW_MAX + 1)
    assert big.score(None, None, k, v, None, {}).shape == (1, 2, 64)
    big.compress(None, None, k, v, None, {})
    assert calls[n:] == [("generic", 32)]


# --------------------------------------------------------------------------------------------------
# the press on tiny Llamas, with the float64 stand-ins in place of the kernels
# --------------------------------------------------------------------------------------------------
@pytest.fixture
def standins(monkeypatch):
    """The float64 stand-ins, with every CUR call recorded as (entry point, S, window, leverage type)."""
    cpu_backend.install(monkeypatch)
    criticalkv_backend.install(monkeypatch)
    calls = []

    def score(keys, values, sinks, leverage_type, window, G=None):
        calls.append(("score", keys.shape[2], window, leverage_type))
        return CB.cur_score(keys, values, sinks, leverage_type, window, G)

    def compress(keys, values, sinks, leverage_type, window, G, n_kept, return_indices=False, return_scores=False):
        calls.append(("compress", keys.shape[2], window, leverage_type))
        return CB.cur_compress(keys, values, sinks, leverage_type, window, G, n_kept, return_indices, return_scores)

    monkeypatch.setattr(native, "cur_score", score)
    monkeypatch.setattr(native, "cur_compress", compress)
    return calls


ALONE = [("kv_product", True, 16), ("kv_avg", True, 7), ("key", False, 16), ("value", True, 16)]


@pytest.mark.parametrize("leverage_type,local,w", ALONE, ids=[f"{t}-{int(loc)}-{w}" for t, loc, w in ALONE])
def test_press_keeps_the_reference_rows(standins, ref, leverage_type, local, w):
    """The press on a float32 tiny Llama keeps the rows the reference's CURPress keeps (150 positions: the last window
    is short)."""
    ids = distinct_ids(150, seed=5)
    options = dict(compression_ratio=0.4, leverage_type=leverage_type, use_local_approximation=local,
                   local_window_size=w)

    def reference(kvpress):
        model, cache = tiny_model(), DynamicCache()
        with kvpress.CURPress(**options)(model):
            model.model(input_ids=ids, past_key_values=cache, cache_position=torch.arange(ids.shape[1]))
        return {"len": cache.get_seq_length(),
                **{f"sig{i}": rows_signature(la.keys, la.values) for i, la in enumerate(cache.layers)}}

    want = ref(f"press/{leverage_type}/{int(local)}/{w}", reference)
    model, cache = tiny_model(), DynamicCache()
    with CURPress(**options)(model):
        model.model(input_ids=ids, past_key_values=cache)
    assert cache.get_seq_length() == int(want["len"]) == 90
    assert standins == [("compress", 150, w if local else 0, leverage_type)] * 2
    for i, la in enumerate(cache.layers):
        close(rows_signature(la.keys, la.values), want[f"sig{i}"], f"layer {i}")


WRAPPED = {
    "chunk": lambda m: m.ChunkPress(m.CURPress(compression_ratio=0.4), chunk_length=40),
    "rerotate": lambda m: m.KeyRerotationPress(m.CURPress(compression_ratio=0.4)),
    "composed": lambda m: m.ComposedPress([m.CURPress(compression_ratio=0.2), m.KnormPress(compression_ratio=0.25)]),
    "critical": lambda m: m.CriticalKVPress(m.CURPress(compression_ratio=0.4)),
}


class _Ours:
    ChunkPress, KeyRerotationPress, ComposedPress, CriticalKVPress = (ChunkPress, KeyRerotationPress, ComposedPress,
                                                                      CriticalKVPress)
    CURPress, KnormPress = CURPress, KnormPress


@pytest.mark.parametrize("wrapper", sorted(WRAPPED))
def test_wrapped_press_keeps_the_reference_rows(standins, ref, wrapper):
    """ChunkPress (chunks of 40: not a multiple of the window, so each chunk has its own windows and a short last one),
    KeyRerotationPress, ComposedPress and CriticalKVPress over CURPress against the same wrappers of the reference."""
    ids = distinct_ids(150, seed=5)

    def reference(kvpress):
        model, cache = tiny_model(), DynamicCache()
        with WRAPPED[wrapper](kvpress)(model):
            model.model(input_ids=ids, past_key_values=cache, cache_position=torch.arange(ids.shape[1]))
        return {"len": cache.get_seq_length(),
                **{f"sig{i}": rows_signature(la.keys, la.values) for i, la in enumerate(cache.layers)}}

    want = ref(f"wrapped/{wrapper}", reference)
    model, cache = tiny_model(), DynamicCache()
    with WRAPPED[wrapper](_Ours)(model):
        model.model(input_ids=ids, past_key_values=cache)
    assert cache.get_seq_length() == int(want["len"])
    if wrapper == "chunk":
        assert standins == ([("score", 40, 16, "kv_product")] * 3 + [("score", 30, 16, "kv_product")]) * 2
    for i, la in enumerate(cache.layers):
        close(rows_signature(la.keys, la.values), want[f"sig{i}"], f"layer {i}")


def test_adakv_decoding_and_a_user_subclass(standins):
    ids = distinct_ids(150, seed=5)
    model, cache = tiny_model(), DynamicCache()
    with AdaKVPress(CURPress(compression_ratio=0.4))(model):
        model.model(input_ids=ids, past_key_values=cache)
    attn = [layer.self_attn for layer in model.model.layers]
    assert cache.get_seq_length() == 150 and standins == [("score", 150, 16, "kv_product")] * 2
    for a, layer in zip(attn, cache.layers):
        b, h, s = a.masked_key_indices
        assert len(b) == 2 * 2 * 60
        # the masked positions are the lowest float64 scores over the heads of each batch row, sinks never among them
        sc = CB.cur_score(layer.keys, layer.values, 4, "kv_product", 16)
        assert (sc[b, h, s] < 1).all() and (s >= 4).all()
        a.masked_key_indices = None

    del standins[:]
    model, cache = tiny_model(), DynamicCache()
    with DecodingPress(CURPress(), compression_interval=4, target_size=100)(model):
        model.model(input_ids=ids[:, :120], past_key_values=cache)
        for t in range(8):
            model.model(input_ids=ids[:, 120 + t:121 + t], past_key_values=cache)
    assert cache.get_seq_length() == 100
    assert standins == [("compress", 124, 16, "kv_product")] * 2 + [("compress", 104, 16, "kv_product")] * 2

    class Reversed(CURPress):
        def score(self, module, hidden_states, keys, values, attentions, kwargs):
            return -super().score(module, hidden_states, keys, values, attentions, kwargs)

    del standins[:]
    model, cache = tiny_model(), DynamicCache()
    with Reversed(compression_ratio=0.4)(model):
        model.model(input_ids=ids, past_key_values=cache)
    # the overriding score() is used: the generic selection, and the sinks (score -1, the lowest) are dropped
    assert cache.get_seq_length() == 90 and standins == [("score", 150, 16, "kv_product")] * 2
