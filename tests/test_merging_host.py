"""MergingPress on the GPU-less box: the C ABI's checks of the two new entry points, the workspace and launch count of the
new scorer id, the argument lists of their wrappers, the float64 definition against the UNMODIFIED reference, and the
press alone and around the scorer presses on float32 tiny Llamas, with the float64 stand-ins of tests/merging_backend.py
in place of the kernels.

Statuses: every argument of kvp_merging_compress / kvp_merging_merge made invalid on its own (or set to another valid
value), and every pair of such changes, against a restatement of the documented check order (include/kvpress_b200.h).
The pointers are fake and never dereferenced: the calls run in a child process that sees no GPU, so a call that passes
every check fails at its first CUDA call with KVP_ERR_CUDA (-6), except a merge call with n_kept == 0, which enqueues
nothing and returns KVP_OK.

Reference: what the reference's `MergingPress.merge` returns on seeded float32 K / V, and the rows its press keeps on
float32 tiny Llamas, are stored in tests/golden/merging_reference.npz. To re-record it from a checkout of the reference
(located as in oracle/build_ref.py):
    KVP_RECORD_MERGING=1 python -m pytest tests/test_merging_host.py
"""
import ctypes
import math
from pathlib import Path

import pytest
import torch
from transformers import DynamicCache

from kvpress_b200 import (ComposedPress, CriticalKVPress, ExpectedAttentionPress, KnormPress, MergingPress,
                          PrefillDecodingPress, PyramidKVPress, ScorerPress, SnapKVPress, native)
from tests import abi_cases, cpu_backend, criticalkv_backend, merging_backend as MB
from tests.abi_cases import GOOD, ODD16
from tests.support import TO_32BIT, close, kv, rec, reference_store, rows_signature  # noqa: F401  (rec: fixture)
from tests.tiny_models import distinct_ids, tiny_model

STORE = Path(__file__).resolve().parent / "golden" / "merging_reference.npz"
ODD4 = GOOD + 2  # 2-byte but not 4-byte aligned


# --------------------------------------------------------------------------------------------------
# C ABI statuses
# --------------------------------------------------------------------------------------------------
def _checks(f, a, compress):
    """target_out / sim_out (and kept_idx) 4-byte alignment -> similarity_threshold -> merge_fraction."""
    ptrs = [a["target"], a["sim"]] + ([] if compress else [a["kept"]])
    if any(x is not None and x % 4 for x in ptrs):
        return -4
    if not 0.0 <= a["thr"] <= 1.0 or not 0.0 < a["frac"] <= 1.0:  # NaN fails both
        return -7
    return 0


ABI = abi_cases.Spec(
    scorer=native.SCORER_MERGING,
    slots={"kvp_merging_compress": "scores sstride K V thr frac K_out V_out idx target sim ws ws_bytes stream",
           "kvp_merging_merge": "K V kept thr frac V_out target sim ws ws_bytes stream"},
    valid=dict(scores=GOOD, sstride="sstride", K=GOOD, V=GOOD, kept=GOOD, thr=0.0, frac=1.0, K_out=GOOD, V_out=GOOD,
               idx=GOOD, target=GOOD, sim=GOOD, ws=GOOD, ws_bytes="enough", stream=0),
    changes={
        "p": {"null": None},
        "dtype": {"1": 1, "3": 3},
        "S": {"0": 0, "1": 1},
        "D": {"8": 8, "12": 12, "264": 264},
        "n_kept": {"-1": -1, "0": 0, "1000": 1000, "1001": 1001},
        "v_stride": {"s100": (256000, 128000, 100)},
        "scores": {"null": None},
        "sstride": {"null": None},
        "K": {"null": None, "odd": ODD16},
        "V": {"null": None, "odd": ODD16},
        "kept": {"null": None, "odd16": ODD16, "odd4": ODD4},
        "thr": {"-0.1": -0.1, "0.5": 0.5, "1": 1.0, "1.5": 1.5, "nan": math.nan},
        "frac": {"0": 0.0, "0.3": 0.3, "1.01": 1.01, "nan": math.nan},
        "K_out": {"null": None, "odd": ODD16},
        "V_out": {"null": None, "odd": ODD16},
        "idx": {"null": None},
        "target": {"null": None, "odd16": ODD16, "odd4": ODD4},
        "sim": {"null": None, "odd4": ODD4},
        "ws": {"null": None, "odd": ODD16},
        "ws_bytes": {"short": "short"},
    },
    operands={"score": (["K", "V", "kept", "V_out"], ["K", "V", "V_out"]), "compress": (["scores", "sstride"], [])},
    checks=_checks, problem=("dtype", "S", "D", "n_kept", "v_stride"))


def test_every_status_of_the_merging_entry_points_follows_the_check_order():
    got = abi_cases.in_child("tests.abi_cases:statuses", __name__)
    want = {}
    for name in ABI.slots:
        for label, c in abi_cases.cases(ABI, name).items():
            st = abi_cases.expected(ABI, name, c)
            n_kept = c.get("n_kept", abi_cases.FIELDS["n_kept"])
            if name == "kvp_merging_merge" and st == -6 and n_kept == 0:
                st = 0  # nothing kept: nothing enqueued
            want[f"{name}({label})"] = st
    assert sorted(got) == sorted(want) and len(got) > 1500
    diffs = [f"{k}: {got[k]} != {want[k]}" for k in want if got[k] != want[k]]
    assert not diffs, f"{len(diffs)} differences, first ones:\n" + "\n".join(diffs[:30])
    assert want["kvp_merging_merge(n_kept=0)"] == 0 and want["kvp_merging_compress(n_kept=0)"] == 0
    assert want["kvp_merging_compress(thr=nan)"] == want["kvp_merging_merge(frac=nan)"] == -7
    assert want["kvp_merging_compress(target=odd4)"] == want["kvp_merging_merge(kept=odd4)"] == -4


def test_workspace_and_launch_count_of_the_new_scorer_id():
    """The merge's workspace is the selection stage's plus, per row and position (S rounded up to 256): the gathered keys
    with head_dim padded to a multiple of 64, and nine 4-byte arrays, each rounded up to 256 bytes. It does not depend
    on n_kept. A compress is 7 launches, 6 when nothing is evicted. The id is 13; 10 and 12 are not assigned."""
    lib = native.load()
    assert native.SCORER_MERGING == 13 and native.SCORER_CUR == 11
    p = native.KvpProblem()
    p.B, p.Hkv, p.Hq, p.dtype = 1, 8, 8, 0
    up = lambda x: -(-x // 256) * 256  # noqa: E731
    for S, D in [(1, 8), (2, 64), (255, 72), (256, 128), (257, 192), (4096, 256), (131072, 128)]:
        for n_kept in (0, S // 2, S):
            p.S, p.D, p.n_kept = S, D, n_kept
            m, generic, n = ctypes.c_size_t(0), ctypes.c_size_t(0), ctypes.c_int(0)
            assert lib.kvp_workspace_bytes(ctypes.byref(p), native.SCORER_MERGING, ctypes.byref(m)) == 0
            assert lib.kvp_workspace_bytes(ctypes.byref(p), native.SCORER_GENERIC, ctypes.byref(generic)) == 0
            rows = 8 * up(S)
            assert m.value == generic.value + up(rows * -(-D // 64) * 64 * 2) + 9 * up(rows * 4)
            assert lib.kvp_launches_per_compress(ctypes.byref(p), native.SCORER_MERGING, ctypes.byref(n)) == 0
            assert n.value == (6 if n_kept == S else 7)
    for unknown in (10, 12):
        assert lib.kvp_launches_per_compress(ctypes.byref(p), unknown, ctypes.byref(n)) == -7


# --------------------------------------------------------------------------------------------------
# wrappers: each argument after the kvp_problem, in order, down to the workspace and the stream
# --------------------------------------------------------------------------------------------------
def test_merging_wrappers_pass_their_full_argument_list(rec):  # noqa: F811
    P = lambda t: t.data_ptr()  # noqa: E731
    k, v = kv(B=2, H=2, S=300, D=64)
    scores = torch.randn(2, 2, 300).bfloat16()

    def last(name, n_kept):
        got, p, a = rec.calls[-1]
        assert got == name and (p["n_kept"], p["Hkv"], p["D"], p["S"]) == (n_kept, 2, 64, 300)
        problem = native.make_problem(k, v, n_kept)
        assert a[-2:] == [native.workspace_bytes(problem, native.SCORER_MERGING), 0] and a[-3] != 0
        return a[:-3]

    k_out, v_out, idx, target, sim = native.merging_compress(scores, k, v, 0.25, 0.75, 100, return_indices=True,
                                                             return_plan=True)
    assert last("kvp_merging_compress", 100) == [P(scores), (600, 300), P(k), P(v), 0.25, 0.75, P(k_out), P(v_out),
                                                 P(idx), P(target), P(sim)]
    assert k_out.shape == v_out.shape == (2, 2, 100, 64) and idx.dtype == target.dtype == torch.int32
    assert target.shape == sim.shape == (2, 2, 200) and sim.dtype == torch.float32
    k_out, v_out, idx, target, sim = native.merging_compress(scores, k, v, 0.0, 1.0, 100)
    assert idx is None and target is None and sim is None
    assert last("kvp_merging_compress", 100)[6:] == [P(k_out), P(v_out), 0, 0, 0]
    kept = torch.arange(0, 300, 3).expand(2, 2, -1)  # int64: cast to int32
    v_out, target, sim = native.merging_merge(k, v, kept, 1.0, 0.5, return_plan=True)
    a = last("kvp_merging_merge", 100)
    assert a[:2] == [P(k), P(v)] and a[2] != 0 and a[3:] == [1.0, 0.5, P(v_out), P(target), P(sim)]
    assert v_out.shape == (2, 2, 100, 64) and target.shape == (2, 2, 200)
    # the gate is checked before anything is enqueued
    n = len(rec.calls)
    for thr, frac in [(-0.1, 1.0), (1.5, 1.0), (math.nan, 1.0), (0.0, 0.0), (0.0, 1.5), (0.0, math.nan)]:
        with pytest.raises(ValueError):
            native.merging_compress(scores, k, v, thr, frac, 100)
    native.merging_compress(scores, k, v, 0.0, 1.0, 0)  # n_kept == 0: nothing is enqueued
    assert len(rec.calls) == n


# --------------------------------------------------------------------------------------------------
# the float64 definition against the unmodified reference
# --------------------------------------------------------------------------------------------------
ref = reference_store(STORE, "KVP_RECORD_MERGING", TO_32BIT)

# (name, thr, frac): the gate's regimes, including the fraction whose quantile falls between two -inf order statistics
GATES = [("t0f1", 0.0, 1.0), ("t0.1f1", 0.1, 1.0), ("t0f0.75", 0.0, 0.75), ("t0.05f0.3", 0.05, 0.3),
         ("t0.3f0.75", 0.3, 0.75)]


def _definition_inputs(kind: str, S: int = 96, n_kept: int = 40):
    g = torch.Generator().manual_seed(S * 7 + n_kept)
    k = torch.randn(2, 2, S, 16, generator=g)
    v = torch.randn(2, 2, S, 16, generator=g)
    scores = torch.randn(2, 2, S, generator=g)
    if kind == "shared":  # a common direction: large similarities, many contributions per kept row
        k = k + 2.0 * torch.randn(2, 2, 1, 16, generator=g)
    idx = scores.topk(n_kept, dim=-1).indices
    if kind == "zero":
        k[0, 0, ::3] = 0
    if kind == "nan":
        k[1, 1, idx[1, 1, 3]] = float("nan")
    return k, v, idx


@pytest.mark.parametrize("kind", ["plain", "shared", "zero", "nan"])
@pytest.mark.parametrize("gate", GATES, ids=[g[0] for g in GATES])
def test_float64_definition_is_the_reference(ref, kind, gate):
    """tests/merging_backend.py against the reference's own merge() on float32 inputs, to float32 rounding: the merged
    kept rows, and the evicted rows untouched."""
    name, thr, frac = gate
    k, v, idx = _definition_inputs(kind)

    def reference(kvpress):
        from kvpress.presses.merging_press import MergingPress as RefMerging

        press = RefMerging(press=kvpress.KnormPress(compression_ratio=0.5), similarity_threshold=thr,
                           merge_fraction=frac)
        keys, values = press.merge(k, v, idx)
        assert keys is k
        return {"values": values}

    want = torch.as_tensor(ref(f"definition/{kind}/{name}", reference)["values"], dtype=torch.float64)
    kept = idx.sort(dim=-1).values
    v64, target, max_sim = MB.merge64(k, v, kept, thr, frac)
    got = v.double().clone()
    got.scatter_(2, kept.unsqueeze(-1).expand(-1, -1, -1, 16), v64)
    nan = want.isnan()
    assert torch.equal(nan, got.isnan())
    close(got[~nan], want[~nan], f"{kind}/{name}")
    if kind == "zero":
        ev = MB.complement(kept, 96)
        zero = (k.gather(2, ev.unsqueeze(-1).expand(-1, -1, -1, 16)) == 0).all(-1)
        assert (target[zero] == 0).all() and (max_sim[zero] == 0).all()
    if kind == "nan":
        assert (target[1, 1] == (kept[1, 1] == idx[1, 1, 3]).nonzero().item()).all() and max_sim[1, 1].isnan().all()


def test_quantile_between_two_minus_inf_statistics_merges_nothing():
    """q = 0.25 over [-inf, -inf, 0.2, 0.5, 0.9]: torch.lerp of two -inf order statistics is NaN, so nothing passes."""
    sim = torch.tensor([[[-0.5, -0.4, 0.2, 0.5, 0.9]]])
    assert not MB.gate(sim, 0.0, 0.75).any()
    assert MB.gate(sim, 0.0, 0.5).tolist() == [[[False, False, True, True, True]]]  # the median, 0.2


def test_press_mirrors_the_reference_fields():
    press = MergingPress(KnormPress(0.25))
    assert (press.similarity_threshold, press.merge_fraction) == (0.0, 1.0)
    assert press.compression_ratio == 0.25
    press.compression_ratio = 0.5
    assert press.press.compression_ratio == 0.5
    with pytest.raises(AssertionError, match="requires a ScorerPress"):
        MergingPress()
    with pytest.raises(AssertionError):
        MergingPress(KnormPress(0.5), similarity_threshold=1.5)
    with pytest.raises(AssertionError, match="merge_fraction"):
        MergingPress(KnormPress(0.5), merge_fraction=0.0)


def test_merge_checks_its_indices(monkeypatch):
    MB.install(monkeypatch)
    k, v, idx = _definition_inputs("plain")
    press = MergingPress(KnormPress(0.5))
    keys, values = press.merge(k, v, idx)
    assert keys is k and values.shape == v.shape
    same = press.merge(k, v, torch.arange(96).expand(2, 2, -1))  # nothing evicted
    assert same[0] is k and same[1] is v
    with pytest.raises(ValueError, match="distinct"):
        press.merge(k, v, torch.zeros(2, 2, 4, dtype=torch.long))
    with pytest.raises(ValueError, match="lie in"):
        press.merge(k, v, torch.full((2, 2, 4), 96))


# --------------------------------------------------------------------------------------------------
# the press on tiny Llamas, with the float64 stand-ins in place of the kernels
# --------------------------------------------------------------------------------------------------
class _UserScores(ScorerPress):
    """A user press with float32 scores of its own."""

    def score(self, module, hidden_states, keys, values, attentions, kwargs):
        return keys.float().sum(dim=-1) - 0.1 * values.float().sum(dim=-1)


def _user(m, r):
    cls = type("UserScores", (m.ScorerPress,), {"score": _UserScores.score})
    return cls(compression_ratio=r)


INNER = {
    "knorm": lambda m: m.KnormPress(compression_ratio=0.5),
    "snapkv": lambda m: m.SnapKVPress(compression_ratio=0.5, window_size=16),
    "ea": lambda m: m.ExpectedAttentionPress(compression_ratio=0.4, use_vnorm=False),
    "critical": lambda m: m.CriticalKVPress(m.KnormPress(compression_ratio=0.5)),
    "pyramid": lambda m: m.PyramidKVPress(compression_ratio=0.5, window_size=16),
    "user": lambda m: _user(m, 0.5),
}
WRAPPED = {
    "composed": lambda m: m.ComposedPress([m.MergingPress(m.KnormPress(compression_ratio=0.3)),
                                           m.KnormPress(compression_ratio=0.2)]),
    "prefill_decoding": lambda m: m.PrefillDecodingPress(prefilling_press=m.MergingPress(
        m.KnormPress(compression_ratio=0.5), merge_fraction=0.75)),
}


class _Ours:
    KnormPress, SnapKVPress, ExpectedAttentionPress, CriticalKVPress, PyramidKVPress = (
        KnormPress, SnapKVPress, ExpectedAttentionPress, CriticalKVPress, PyramidKVPress)
    ScorerPress, ComposedPress, PrefillDecodingPress, MergingPress = (ScorerPress, ComposedPress, PrefillDecodingPress,
                                                                      MergingPress)


def _run(make, kvpress, model, ids, record: bool):
    cache = DynamicCache()
    with make(kvpress)(model):
        if record:
            model.model(input_ids=ids, past_key_values=cache, cache_position=torch.arange(ids.shape[1]))
        else:
            model.model(input_ids=ids, past_key_values=cache)
    return {"len": cache.get_seq_length(),
            **{f"keys{i}": rows_signature(la.keys, 0 * la.values) for i, la in enumerate(cache.layers)},
            **{f"sig{i}": rows_signature(la.keys, la.values) for i, la in enumerate(cache.layers)}}


@pytest.mark.parametrize("name", sorted(INNER) + sorted(WRAPPED))
def test_press_keeps_the_reference_rows_and_values(monkeypatch, ref, name):
    """The press (around each scorer, or inside a wrapper) on a float32 tiny Llama keeps the reference's rows: its keys
    exactly as gathered, its values merged to float32 rounding."""
    cpu_backend.install(monkeypatch)
    criticalkv_backend.install(monkeypatch)
    MB.install(monkeypatch)
    model, ids = tiny_model(), distinct_ids(150, seed=5)
    if name in INNER:
        make = lambda m: m.MergingPress(INNER[name](m), similarity_threshold=0.05)  # noqa: E731
    else:
        make = WRAPPED[name]
    want = ref(f"press/{name}", lambda kvpress: _run(make, kvpress, model, ids, True))
    got = _run(make, _Ours, model, ids, False)
    assert got["len"] == int(want["len"])
    if name in ("knorm", "critical", "pyramid", "user", "prefill_decoding"):
        assert got["len"] == 75  # the reference's uniform int(k_len * (1 - ratio)), PyramidKV's per-layer count unused
    for i in range(2):
        close(got[f"keys{i}"], want[f"keys{i}"], f"keys of layer {i}")
        close(got[f"sig{i}"], want[f"sig{i}"], f"layer {i}")


def test_reference_properties_on_a_tiny_llama(monkeypatch):
    """The four properties of the reference's tests/presses/test_merging_press.py on a batch of two prompts: merged
    values differ from hard eviction, keys are unchanged, the merged rows carry information of the evicted ones (each
    hard-evicted row equals its uncompressed row, a merged one does not), and the batch keeps its shape."""
    cpu_backend.install(monkeypatch)
    MB.install(monkeypatch)
    model, ids = tiny_model(), distinct_ids(64, seed=42)

    def prefill(press):
        cache = DynamicCache()
        if press is None:
            model.model(input_ids=ids, past_key_values=cache)
            return cache
        with press(model):
            model.model(input_ids=ids, past_key_values=cache)
        return cache

    full = prefill(None)
    for ratio in (0.5, 0.7):
        hard, merged = prefill(KnormPress(ratio)), prefill(MergingPress(KnormPress(ratio)))
        assert hard.get_seq_length() == merged.get_seq_length() == int(64 * (1 - ratio))
        assert any(not torch.equal(a.values, b.values) for a, b in zip(hard.layers, merged.layers))
        assert all(torch.equal(a.keys, b.keys) for a, b in zip(hard.layers, merged.layers))

        def error(cache):
            total = 0.0
            for f, la in zip(full.layers, cache.layers):  # each kept row against its own uncompressed row
                match = (la.keys[..., :, None, :] == f.keys[..., None, :, :]).all(-1).float().argmax(-1)
                total += (la.values - f.values.gather(2, match.unsqueeze(-1).expand_as(la.values))).norm().item()
            return total

        if ratio == 0.7:
            assert error(merged) > 0 and error(hard) == 0  # merged rows carry the evicted information
    assert ids.shape[0] == 2 and all(la.keys.shape[0] == 2 for la in merged.layers)  # a batch of two prompts
