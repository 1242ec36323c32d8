"""ThinK on the GPU-less box: the C ABI's checks of kvp_think_prune, the workspace and launch count of scorer id 14,
the wrapper's argument list, the float64 definition against the UNMODIFIED reference, and the press alone and inside
ComposedPress / PrefillDecodingPress on tiny float32 Llamas with the float64 stand-in (tests/think_backend.py) in place
of the kernel.

Statuses: every argument of kvp_think_prune made invalid on its own (or set to another valid value), and every pair of
such changes to two different arguments, against a restatement of the documented check order (include/kvpress_b200.h).
The pointers are fake, 16-byte aligned or not, and never dereferenced: the calls run in a child process that sees no
GPU, so a call that passes every check fails at its first CUDA call with KVP_ERR_CUDA (-6).

Reference: what the reference's `ThinKPress.compress` returns, and the channel scores it hands to `topk`, on seeded
float32 keys and window queries, and what the reference's presses leave in the cache of a tiny Llama, are stored in
tests/golden/think_reference.npz. To re-record them from a checkout of the reference (located as in oracle/build_ref.py):
    KVP_RECORD_THINK=1 python -m pytest tests/test_think_host.py
"""
import ctypes
from pathlib import Path
from types import SimpleNamespace

import pytest
import torch
from transformers import DynamicCache

from kvpress_b200 import (ComposedPress, KnormPress, PrefillDecodingPress, SnapKVPress, ThinKPress, native)
from kvpress_b200.presses.adakv_press import AdaKVPress
from tests import abi_cases, cpu_backend, think_backend as TB
from tests.abi_cases import GOOD, ODD16
from tests.support import TO_32BIT, close, kv, rec, reference_store, rows_signature  # noqa: F401  (rec: fixture)
from tests.tiny_models import distinct_ids, tiny_model

STORE = Path(__file__).resolve().parent / "golden" / "think_reference.npz"
ODD4 = 0x10002  # 2-byte but not 4-byte aligned


# --------------------------------------------------------------------------------------------------
# C ABI statuses
# --------------------------------------------------------------------------------------------------
def expected(c: dict) -> int:
    """The documented check order of kvp_think_prune: p null -> validate (K's strides in place of v_stride) ->
    window >= 1 and 0 <= n_pruned <= D -> n_pruned == 0 returns KVP_OK -> K, q null -> K, q 16-byte and the outputs
    4-byte alignment -> workspace null -> alignment -> size."""
    f = {**abi_cases.FIELDS, **{k: v for k, v in c.items() if k in abi_cases.FIELDS}}
    a = {**ABI_VALID, **{k: v for k, v in c.items() if k not in abi_cases.FIELDS}}
    if c.get("p", 0) is None:
        return -1
    rc = abi_cases.validate({k: v for k, v in c.items() if k != "v_stride"}, f)
    if rc:
        return rc
    if a["window"] < 1 or not 0 <= a["n_pruned"] <= f["D"]:
        return -7
    if a["n_pruned"] == 0:
        return 0
    if a["K"] is None or a["q"] is None:
        return -1
    if a["K"] % 16 or a["q"] % 16 or any(x is not None and x % 4 for x in (a["pruned"], a["scores"])):
        return -4
    if a["ws"] is None:
        return -1
    if a["ws"] % 16:
        return -4
    return -5 if a["ws_bytes"] == "short" else -6


SLOTS = "K q window n_pruned pruned scores ws ws_bytes stream"
ABI_VALID = dict(K=GOOD, q=GOOD, window=32, n_pruned=64, pruned=GOOD, scores=GOOD, ws=GOOD, ws_bytes="enough",
                 stream=0)
ABI_CHANGES = {
    "p": {"null": None},
    "dtype": {"1": 1, "3": 3},
    "S": {"0": 0, "1": 1},
    "D": {"8": 8, "12": 12, "64": 64, "264": 264},
    "Hq": {"5": 5, "8": 8},
    "n_kept": {"-1": -1, "0": 0, "1001": 1001},
    "k_stride": {"s100": (256000, 128000, 100)},
    "v_stride": {"s100": (256000, 128000, 100)},  # ignored
    "K": {"null": None, "odd": ODD16},
    "q": {"null": None, "odd": ODD16},
    "window": {"0": 0, "-1": -1, "1": 1, "257": 257},
    "n_pruned": {"-1": -1, "0": 0, "1": 1, "128": 128, "129": 129},
    "pruned": {"null": None, "odd": ODD4},
    "scores": {"null": None, "odd": ODD4},
    "ws": {"null": None, "odd": ODD16},
    "ws_bytes": {"short": "short"},
}


def think_cases() -> dict:
    return abi_cases.case_matrix({s: ABI_CHANGES.get(s, {}) for s in
                                  ["p", "dtype", "S", "D", "Hq", "n_kept", "k_stride", "v_stride", *SLOTS.split()]})


def think_statuses() -> dict:
    """The library's status of every case. Run only in a process that sees no GPU."""
    nat, lib = abi_cases.load_native()
    out = {}
    for label, c in think_cases().items():
        pr = None if c.get("p", 0) is None else abi_cases.problem(nat, c, abi_cases.FIELDS)
        args = [None if pr is None else ctypes.byref(pr)]
        for slot in SLOTS.split():
            v = c.get(slot, ABI_VALID[slot])
            if v in ("enough", "short"):
                v = abi_cases.workspace_bytes(lib, pr, nat.SCORER_THINK) - (v == "short")
            args.append(v)
        out[label] = lib.kvp_think_prune(*args)
    return out


def test_every_status_of_kvp_think_prune_follows_the_check_order():
    got = abi_cases.in_child("tests.test_think_host:think_statuses")
    want = {label: expected(c) for label, c in think_cases().items()}
    assert sorted(got) == sorted(want) and len(got) > 600
    diffs = [f"{k}: {got[k]} != {want[k]}" for k in want if got[k] != want[k]]
    assert not diffs, f"{len(diffs)} differences, first ones:\n" + "\n".join(diffs[:30])
    assert got["valid"] == -6 and got["n_pruned=0"] == 0 and got["v_stride=s100"] == -6


def _problem(**kw):
    p = native.KvpProblem()
    p.B, p.Hkv, p.Hq, p.S, p.D, p.n_kept, p.dtype = 1, 8, 32, 4096, 128, 4096, 0
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def test_workspace_formula_and_launch_count_of_scorer_14():
    """Tickets, the bitmask and one fp32 partial per channel and 256-position block, each region rounded up to 256
    bytes; monotone in S. A call is 3 launches. Ids 10 and 12 stay unknown."""
    lib = native.load()
    assert native.SCORER_THINK == 14
    a256 = lambda x: -(-x // 256) * 256  # noqa: E731
    last = 0
    for B, H, D in [(1, 8, 128), (2, 3, 8), (4, 2, 256)]:
        last = 0
        for S in (1, 255, 256, 257, 4099, 32768, 131072):
            p = _problem(B=B, Hkv=H, Hq=H, S=S, D=D, n_kept=S)
            out, n = ctypes.c_size_t(0), ctypes.c_int(0)
            assert lib.kvp_workspace_bytes(ctypes.byref(p), native.SCORER_THINK, ctypes.byref(out)) == 0
            R = B * H
            assert out.value == a256(4 * R) + a256(32 * R) + a256(4 * R * (-(-S // 256)) * D)
            assert out.value >= last
            last = out.value
            assert lib.kvp_launches_per_compress(ctypes.byref(p), native.SCORER_THINK, ctypes.byref(n)) == 0
            assert n.value == 3
    p = _problem()
    n = ctypes.c_int(0)
    for unknown in (10, 12, 15):
        assert lib.kvp_launches_per_compress(ctypes.byref(p), unknown, ctypes.byref(n)) == -7


# --------------------------------------------------------------------------------------------------
# the wrapper: each argument after the kvp_problem, in order, down to the workspace and the stream
# --------------------------------------------------------------------------------------------------
def test_think_prune_passes_its_full_argument_list(rec):  # noqa: F811
    P = lambda t: t.data_ptr()  # noqa: E731
    k, _ = kv(B=2, H=2, S=300, D=64)
    q = torch.randn(2, 8, 32, 64).to(k.dtype)
    out, pruned, scores = native.think_prune(k, q, 16, return_pruned=True, return_scores=True)
    got, p, a = rec.calls[-1]
    assert got == "kvp_think_prune" and out is k
    assert (p["n_kept"], p["Hq"], p["Hkv"], p["D"], p["S"]) == (300, 8, 2, 64, 300)
    assert p["k_stride"] == p["v_stride"] == (2 * 300 * 64, 300 * 64, 64)
    ws = native.workspace_bytes(native.make_problem(k, k, 300, 8), native.SCORER_THINK)
    assert a[:6] == [P(k), P(q), 32, 16, P(pruned), P(scores)] and a[-2:] == [ws, 0] and a[-3] != 0
    assert pruned.shape == (2, 2, 16) and pruned.dtype == torch.int32
    assert scores.shape == (2, 2, 64) and scores.dtype == torch.float32
    _, pruned, scores = native.think_prune(k, q[:, :, :5], 1)
    assert rec.calls[-1][2][2:6] == [5, 1, 0, 0] and pruned is None and scores is None
    # a slice of a longer cache is pruned in place, with its own strides
    ks = k[:, :, 8:-4]
    native.think_prune(ks, q, 3)
    got, p, a = rec.calls[-1]
    assert a[0] == P(ks) and p["S"] == 288 and p["k_stride"] == (2 * 300 * 64, 300 * 64, 64)
    # n_pruned == 0: nothing is enqueued
    n = len(rec.calls)
    assert native.think_prune(k, q, 0, True, True) == (k, None, None)
    assert len(rec.calls) == n
    with pytest.raises(ValueError):
        native.think_prune(k, q, 65)
    with pytest.raises(RuntimeError, match="in place"):
        native.think_prune(k.transpose(2, 3).contiguous().transpose(2, 3), q, 3)
    with pytest.raises(RuntimeError, match="q_window"):
        native.think_prune(k, q[:, :3], 3)
    assert len(rec.calls) == n


# --------------------------------------------------------------------------------------------------
# the float64 definition against the unmodified reference
# --------------------------------------------------------------------------------------------------
ref = reference_store(STORE, "KVP_RECORD_THINK", TO_32BIT)

# (name, B, Hkv, Hq, S, D, w, ratio)
DEFINITION = [
    ("g4", 2, 2, 8, 70, 16, 8, 0.5),
    ("g1", 1, 3, 3, 33, 32, 4, 0.25),
    ("g8-w1", 1, 2, 16, 50, 64, 1, 0.75),
    ("all", 1, 2, 4, 20, 8, 3, 1.0),
    ("one", 2, 1, 2, 40, 24, 5, 0.05),
]


def _definition_inputs(B, Hkv, Hq, S, D, w):
    g = torch.Generator().manual_seed(B * 1000 + Hq * 100 + S + D + w)
    keys = torch.randn(B, Hkv, S, D, generator=g) * torch.rand(D, generator=g) * 2
    q = torch.randn(B, Hq, w, D, generator=g) * (0.5 + torch.rand(D, generator=g))
    return keys, q


@pytest.mark.parametrize("name,B,Hkv,Hq,S,D,w,ratio", DEFINITION, ids=[d[0] for d in DEFINITION])
def test_float64_definition_is_the_reference(ref, name, B, Hkv, Hq, S, D, w, ratio):
    """The float64 stand-in against the reference's own compress() on float32 inputs: the channel scores it ranks (to
    float32 rounding), the pruned set and the keys it returns (exactly)."""
    keys, q = _definition_inputs(B, Hkv, Hq, S, D, w)

    def reference(kvpress):
        from kvpress.presses.think_press import ThinKPress as RefThinK

        press = RefThinK(key_channel_compression_ratio=ratio, window_size=w)
        press.compute_window_queries = lambda *a: q
        module = SimpleNamespace(config=SimpleNamespace(num_attention_heads=Hq), head_dim=D)
        seen = {}
        topk = torch.Tensor.topk

        def spy(t, *a, **kw):
            seen["scores"] = t.clone()
            out = topk(t, *a, **kw)
            seen["pruned"] = out.indices.sort(dim=-1).values
            return out

        torch.Tensor.topk = spy
        try:
            k_ref = keys.clone()
            out, _ = press.compress(module, None, k_ref, None, None, {"hidden_states": None,
                                                                    "position_embeddings": None})
        finally:
            torch.Tensor.topk = topk
        assert out is k_ref
        return {"keys": out, "scores": seen["scores"], "pruned": seen["pruned"]}

    want = ref(f"definition/{name}", reference)
    n_pruned = int(D * ratio)
    close(TB.scores64(keys, q), want["scores"], name)
    got_keys, pruned, scores = TB.think_prune64(keys.clone(), q, n_pruned, True, True)
    assert torch.equal(pruned.long(), torch.as_tensor(want["pruned"]).long())
    assert torch.equal(got_keys, torch.as_tensor(want["keys"]))


def test_stand_in_tie_and_nan_rules():
    """Equal scores keep the lower channel, NaN is pruned last and NaNs go by channel; pruned channels become +0."""
    s = torch.tensor([[[1.0, 2.0, 1.0, float("nan"), 0.5, float("nan"), 2.0, 1.0]]])
    order = [4, 7, 2, 0, 6, 1, 5, 3]  # pruned first .. last
    for n in range(9):
        mask = TB.pruned_mask(s, n)
        assert mask[0, 0].nonzero().flatten().tolist() == sorted(order[:n])
    k = -torch.ones(1, 1, 3, 8)
    q = torch.ones(1, 1, 1, 8)
    q[..., 2] = 0  # channel 2 scores 0
    TB.think_prune64(k, q, 1)
    assert torch.equal(k[..., 2], torch.zeros(1, 1, 3)) and not torch.signbit(k[..., 2]).any()
    assert (k[..., [0, 1, 3, 4, 5, 6, 7]] == -1).all()


# --------------------------------------------------------------------------------------------------
# the press on tiny Llamas, with the float64 stand-ins in place of the kernels
# --------------------------------------------------------------------------------------------------
PRESSES = {
    "alone": lambda m: m.ThinKPress(key_channel_compression_ratio=0.5, window_size=16),
    "short-prompt": lambda m: m.ThinKPress(key_channel_compression_ratio=0.25, window_size=4096),
    "knorm-think": lambda m: m.ComposedPress([m.KnormPress(compression_ratio=0.5),
                                              m.ThinKPress(key_channel_compression_ratio=0.5)]),
    "think-knorm": lambda m: m.ComposedPress([m.ThinKPress(key_channel_compression_ratio=0.5),
                                              m.KnormPress(compression_ratio=0.5)]),
    "snapkv-think": lambda m: m.ComposedPress([m.SnapKVPress(compression_ratio=0.5, window_size=16),
                                               m.ThinKPress(key_channel_compression_ratio=0.5)]),
    "think-snapkv": lambda m: m.ComposedPress([m.ThinKPress(key_channel_compression_ratio=0.5),
                                               m.SnapKVPress(compression_ratio=0.5, window_size=16)]),
    "prefill_decoding": lambda m: m.PrefillDecodingPress(
        prefilling_press=m.ThinKPress(key_channel_compression_ratio=0.75, window_size=8)),
}


PRUNED = {"alone": 0.5, "short-prompt": 0.25, "prefill_decoding": 0.75}  # of the channels; the others 0.5
PRUNED = {name: PRUNED.get(name, 0.5) for name in PRESSES}


class _Ours:
    ThinKPress, KnormPress, SnapKVPress, ComposedPress, PrefillDecodingPress = (
        ThinKPress, KnormPress, SnapKVPress, ComposedPress, PrefillDecodingPress)


def _run(make, kvpress, model, ids, record: bool):
    cache = DynamicCache()
    press = make(kvpress)
    with press(model):
        if record:
            model.model(input_ids=ids, past_key_values=cache, cache_position=torch.arange(ids.shape[1]))
        else:
            model.model(input_ids=ids, past_key_values=cache)
    out = {"len": cache.get_seq_length(), "ratio": getattr(press, "compression_ratio", -1.0)}
    for i, la in enumerate(cache.layers):
        # row order differs after a sequence press (ascending positions here, score order in the reference)
        out[f"zeroed{i}"] = (la.keys == 0).all(dim=2)
        out[f"keys{i}"] = rows_signature(la.keys, 0 * la.values)
        out[f"sig{i}"] = rows_signature(la.keys, la.values)
    return out


@pytest.mark.parametrize("name", sorted(PRESSES))
def test_press_leaves_the_reference_cache(monkeypatch, ref, name):
    """The press alone, composed with Knorm and SnapKV in both orders and as PrefillDecodingPress's prefilling press, on
    a float32 tiny Llama: the same cache length, the same zeroed channels and the same keys and values as the
    reference, to float32 rounding."""
    cpu_backend.install(monkeypatch)
    TB.install(monkeypatch)
    model, ids = tiny_model(), distinct_ids(120, seed=3)
    want = ref(f"press/{name}", lambda kvpress: _run(PRESSES[name], kvpress, model, ids, True))
    got = _run(PRESSES[name], _Ours, model, ids, False)
    assert got["len"] == int(want["len"])
    if name != "prefill_decoding":
        assert got["ratio"] == pytest.approx(float(want["ratio"]))
    for i in range(2):
        zeroed = torch.as_tensor(want[f"zeroed{i}"])
        assert torch.equal(got[f"zeroed{i}"], zeroed), f"zeroed channels of layer {i}"
        assert (zeroed.sum(-1) == int(16 * PRUNED[name])).all()
        close(got[f"keys{i}"], want[f"keys{i}"], f"keys of layer {i}")
        close(got[f"sig{i}"], want[f"sig{i}"], f"layer {i}")


def test_press_prunes_in_place_and_returns_the_same_tensors(monkeypatch):
    TB.install(monkeypatch)
    calls = []
    monkeypatch.setattr(native, "think_prune", lambda *a, **k: calls.append(a) or TB.think_prune64(*a, **k))
    model = tiny_model()
    attn = model.model.layers[0].self_attn
    hidden = torch.randn(1, 10, model.config.hidden_size)
    pos = model.model.rotary_emb(hidden, torch.arange(10).unsqueeze(0))
    keys, values = torch.randn(1, 2, 10, 16), torch.randn(1, 2, 10, 16)
    kw = {"hidden_states": hidden, "position_embeddings": pos}
    k2, v2 = ThinKPress(0.5).compress(attn, hidden, keys, values, None, kw)
    assert k2 is keys and v2 is values and len(calls) == 1
    assert calls[0][1].shape == (1, 4, 10, 16) and calls[0][2] == 8  # a 10-position prompt uses all 10 window rows
    assert (keys == 0).all(dim=2).sum() == 2 * 8
    before = keys.clone()
    assert ThinKPress(0.0).compress(attn, hidden, keys, values, None, kw) == (keys, values)
    assert len(calls) == 1 and torch.equal(keys, before)  # a ratio of 0 launches nothing


def test_compression_ratio_property_and_fields():
    press = ThinKPress()
    assert (press.key_channel_compression_ratio, press.window_size) == (0.0, 32)
    assert ThinKPress(0.5).compression_ratio == 0.25
    with pytest.raises(AttributeError, match="cannot be set"):
        press.compression_ratio = 0.3
    for bad in (-0.1, 1.5, float("nan")):
        with pytest.raises(ValueError):
            ThinKPress(bad)
    with pytest.raises(AssertionError, match="ScorerPress"):
        AdaKVPress(ThinKPress(0.5))
