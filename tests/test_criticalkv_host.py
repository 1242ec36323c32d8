"""CriticalKV on the GPU-less box: the C ABI's checks of the two new entry points, the argument lists of their
wrappers, and the presses against the UNMODIFIED reference through the oracle-backed stand-ins.

Statuses: every argument of kvp_criticalkv_score / kvp_criticalkv_compress made invalid on its own (or set to another
valid value), and every pair of such changes to two different arguments, against a restatement of the documented check
order (include/kvpress_b200.h). The pointers are fake, 16-byte aligned or not, and never dereferenced: the calls run in a
child process that sees no GPU, so a call that passes every check fails at its first CUDA call with KVP_ERR_CUDA (-6).

Reference: what the reference's CriticalKVPress / CriticalAdaKVPress compute on the seeded tiny models is stored in
tests/golden/criticalkv_reference.npz. To re-record it from a checkout of the reference (located as in
oracle/build_ref.py):  KVP_RECORD_CRITICALKV=1 python -m pytest tests/test_criticalkv_host.py
"""
import ctypes
from pathlib import Path

import numpy as np
import pytest
import torch
from transformers import DynamicCache

from kvpress_b200 import (CriticalAdaKVPress, CriticalKVPress, DecodingPress, ExpectedAttentionPress, KnormPress,
                          PrefillDecodingPress, SnapKVPress, native)
from tests import abi_cases, cpu_backend, criticalkv_backend
from tests.abi_cases import GOOD, ODD16
from tests.support import TO_32BIT, close, kv, rec, reference_store, rows_signature  # noqa: F401  (rec: fixture)
from tests.tiny_models import distinct_ids, tiny_model

STORE = Path(__file__).resolve().parent / "golden" / "criticalkv_reference.npz"

# --------------------------------------------------------------------------------------------------
# C ABI statuses
# --------------------------------------------------------------------------------------------------
ODD2 = 0x10001


def _checks(f, a, compress):
    """base_scores 2-byte aligned -> hidden -> wo_stride -> n_first."""
    if a["base"] % 2:
        return -4
    if a["hidden"] <= 0:
        return -7
    if a["wo_stride"] % 8 or a["wo_stride"] < f["Hq"] * f["D"]:
        return -4
    return -7 if not 0 <= a["n_first"] <= (f["n_kept"] if compress else f["S"]) else 0


ABI = abi_cases.Spec(
    scorer=native.SCORER_CRITICALKV,  # Hq * D = 512
    slots={"kvp_criticalkv_score": "V base sstride wo hidden wo_stride eps n_first scores ws ws_bytes stream",
           "kvp_criticalkv_compress": "K V base sstride wo hidden wo_stride eps n_first K_out V_out idx scores ws "
                                      "ws_bytes stream"},
    valid=dict(K=GOOD, V=GOOD, base=GOOD, sstride="sstride", wo=GOOD, hidden=4096, wo_stride=512, eps=1e-4,
               n_first=100, K_out=GOOD, V_out=GOOD, idx=GOOD, scores=GOOD, ws=GOOD, ws_bytes="enough", stream=0),
    changes={
        "p": {"null": None},
        "dtype": {"3": 3},
        "S": {"0": 0},
        "D": {"12": 12, "64": 64},
        "Hq": {"5": 5},
        "n_kept": {"-1": -1, "0": 0, "1000": 1000},
        "v_stride": {"s100": (256000, 128000, 100)},
        "K": {"null": None, "odd": ODD16},
        "V": {"null": None, "odd": ODD16},
        "base": {"null": None, "odd": ODD2, "4-aligned": ODD16},
        "sstride": {"null": None},
        "wo": {"null": None, "odd": ODD16},
        "hidden": {"0": 0, "-1": -1, "1": 1},
        "wo_stride": {"100": 100, "504": 504, "520": 520},
        "n_first": {"-1": -1, "0": 0, "500": 500, "501": 501, "1000": 1000, "1001": 1001},
        "K_out": {"null": None},
        "V_out": {"null": None, "odd": ODD16},
        "idx": {"null": None},
        "scores": {"null": None},
        "ws": {"null": None, "odd": ODD16},
        "ws_bytes": {"short": "short"},
    },
    operands={"score": (["V", "base", "sstride", "wo", "scores"], ["V", "wo"]),
              "compress": (["base", "sstride", "wo"], ["wo"])},
    checks=_checks)


def test_every_status_of_the_criticalkv_entry_points_follows_the_check_order():
    abi_cases.assert_statuses(__name__, 1000)


def test_workspace_and_launch_count_of_the_new_scorer_id():
    lib = native.load()
    p = native.KvpProblem()
    p.B, p.Hkv, p.Hq, p.S, p.D, p.n_kept, p.dtype = 1, 8, 32, 131072, 128, 65536, 0
    ckv, generic, n = ctypes.c_size_t(0), ctypes.c_size_t(0), ctypes.c_int(0)
    assert lib.kvp_workspace_bytes(ctypes.byref(p), native.SCORER_CRITICALKV, ctypes.byref(ckv)) == 0
    assert lib.kvp_workspace_bytes(ctypes.byref(p), native.SCORER_GENERIC, ctypes.byref(generic)) == 0
    assert ckv.value - generic.value >= 8 * 131072 * (4 + 2)  # stage-1 positions and the final scores
    assert lib.kvp_launches_per_compress(ctypes.byref(p), native.SCORER_CRITICALKV, ctypes.byref(n)) == 0
    assert n.value == 8


# --------------------------------------------------------------------------------------------------
# wrappers: each argument after the kvp_problem, in order, down to the workspace and the stream
# --------------------------------------------------------------------------------------------------
def test_criticalkv_wrappers_pass_their_full_argument_list(rec, monkeypatch):  # noqa: F811
    workspaces = []
    real_workspace = native._workspace

    def spy(p, scorer, device):
        workspaces.append((scorer, real_workspace(p, scorer, device)))
        return workspaces[-1][1]

    monkeypatch.setattr(native, "_workspace", spy)
    P = lambda t: t.data_ptr()  # noqa: E731
    k, v = kv(B=2, H=2, S=64, D=64)
    wo = torch.randn(96, 8 * 64 + 16).to(torch.bfloat16)[:, 8:8 + 8 * 64]  # sliced rows: consumed in place
    base = torch.rand(2, 2, 64).to(torch.bfloat16)

    def last(name, n_kept):
        got, p, a = rec.calls[-1]
        assert got == name and (p["n_kept"], p["Hq"], p["D"]) == (n_kept, 8, 64)
        s, ws = workspaces[-1]
        problem = native.make_problem(k, v, n_kept, 8)
        assert s == native.SCORER_CRITICALKV
        assert a[-3:] == [ws.data_ptr(), native.workspace_bytes(problem, native.SCORER_CRITICALKV), 0]
        return a[:-3]

    sc = native.criticalkv_score(base, v, wo, 0.25, 7)
    a = last("kvp_criticalkv_score", 0)
    assert a == [P(v), P(base), (128, 64), P(wo), 96, 8 * 64 + 16, 0.25, 7, P(sc)] and isinstance(a[6], float)
    k_out, v_out, idx, sc = native.criticalkv_compress(base, k, v, wo, 0.5, 10, 20, return_indices=True,
                                                       return_scores=True)
    assert last("kvp_criticalkv_compress", 20) == \
        [P(k), P(v), P(base), (128, 64), P(wo), 96, 8 * 64 + 16, 0.5, 10, P(k_out), P(v_out), P(idx), P(sc)]
    k_out, v_out, idx, sc = native.criticalkv_compress(base.float(), k, v, wo.float(), 0.5, 0, 20)
    a = last("kvp_criticalkv_compress", 20)
    assert a[2] != P(base) and a[5:9] == [96, 8 * 64, 0.5, 0] and a[11:] == [0, 0]  # cast copies, contiguous wo
    with pytest.raises(RuntimeError, match="o_proj.weight"):
        native.criticalkv_score(base, v, wo[:, :100], 0.25, 7)


# --------------------------------------------------------------------------------------------------
# presses against the unmodified reference (CPU stand-ins)
# --------------------------------------------------------------------------------------------------
ref = reference_store(STORE, "KVP_RECORD_CRITICALKV", TO_32BIT)


INNER = {
    "knorm": (lambda m, r: m.KnormPress(compression_ratio=r), lambda r: KnormPress(compression_ratio=r)),
    "snapkv": (lambda m, r: m.SnapKVPress(compression_ratio=r, window_size=16),
               lambda r: SnapKVPress(compression_ratio=r, window_size=16)),
    "ea": (lambda m, r: m.ExpectedAttentionPress(compression_ratio=r, use_vnorm=False),
           lambda r: ExpectedAttentionPress(compression_ratio=r, use_vnorm=False)),
}


@pytest.mark.parametrize("inner", ["knorm", "snapkv", "ea"])
@pytest.mark.parametrize("ratio", [0.25, 0.5, 0.7])
@pytest.mark.parametrize("family", ["llama", "qwen3"])
def test_criticalkv_keeps_the_reference_rows(monkeypatch, ref, inner, ratio, family):
    if inner == "knorm" and family == "qwen3":
        pytest.skip("Qwen3's k_norm makes every key norm (nearly) equal: stage 1 would pick among exact ties, which "
                    "torch.topk and the lowest-position rule break differently")
    cpu_backend.install(monkeypatch)
    criticalkv_backend.install(monkeypatch)
    model, ids = tiny_model(family), distinct_ids(160, seed=5)
    ref_inner, our_inner = INNER[inner]

    def reference(kvpress):
        cache = DynamicCache()
        with kvpress.CriticalKVPress(ref_inner(kvpress, ratio))(model):
            model.model(input_ids=ids, past_key_values=cache, cache_position=torch.arange(ids.shape[1]))
        return {"len": cache.get_seq_length(), **{f"sig{i}": rows_signature(la.keys, la.values)
                                                   for i, la in enumerate(cache.layers)}}

    want = ref(f"critical/{inner}/{ratio}/{family}", reference)
    ours = DynamicCache()
    with CriticalKVPress(our_inner(ratio))(model):
        model.model(input_ids=ids, past_key_values=ours)
    assert ours.get_seq_length() == int(want["len"]) == int(ids.shape[1] * (1 - ratio))
    for i, la in enumerate(ours.layers):
        close(rows_signature(la.keys, la.values), want[f"sig{i}"], f"layer {i}")


def _masks(model, clear=True):
    out = {}
    for i, layer in enumerate(model.model.layers):
        b, h, s = layer.self_attn.masked_key_indices
        order = np.lexsort((s.numpy(), h.numpy(), b.numpy()))
        out[f"mask{i}"] = np.stack([b.numpy()[order], h.numpy()[order], s.numpy()[order]])
        if clear:
            layer.self_attn.masked_key_indices = None
    return out


@pytest.mark.parametrize("inner", ["snapkv", "ea"])
@pytest.mark.parametrize("alpha", [0.0, 0.2, 1.0])
@pytest.mark.parametrize("family", ["llama", "qwen3"])
def test_critical_adakv_masks_and_decoding_step_match_the_reference(monkeypatch, ref, inner, alpha, family):
    cpu_backend.install(monkeypatch)
    criticalkv_backend.install(monkeypatch)
    # one sequence: the reference sums the head budgets over the batch and asks torch.topk for more than S positions
    # once a head's budget exceeds S (criticalkv_press.py:163-176)
    model, ids = tiny_model(family), distinct_ids(160, seed=5)[:1]
    ref_inner, our_inner = INNER[inner]
    nxt = torch.tensor([[7]])

    def reference(kvpress):
        cache = DynamicCache()
        press = kvpress.CriticalAdaKVPress(ref_inner(kvpress, 0.5), alpha_safeguard=alpha)
        with press(model):
            model.model(input_ids=ids, past_key_values=cache, cache_position=torch.arange(ids.shape[1]))
            step = model(input_ids=nxt, past_key_values=cache,
                         cache_position=torch.tensor([ids.shape[1]])).logits
        return {**_masks(model), "logits": step}

    want = ref(f"critical_ada/{inner}/{alpha}/{family}", reference)
    cache = DynamicCache()
    with CriticalAdaKVPress(our_inner(0.5), alpha_safeguard=alpha)(model):
        model.model(input_ids=ids, past_key_values=cache)
        got = _masks(model, clear=False)
        step = model(input_ids=nxt, past_key_values=cache).logits
    for i in range(len(model.model.layers)):
        assert np.array_equal(got[f"mask{i}"], want[f"mask{i}"]), f"layer {i}"
    close(step, want["logits"], "decoding step")
    for layer in model.model.layers:
        layer.self_attn.masked_key_indices = None


def test_prefill_decoding_press_of_the_reference_readme(monkeypatch, ref):
    """PrefillDecodingPress(CriticalKVPress(KnormPress(0.5)), DecodingPress(KnormPress(), 5, 64)) at tiny size."""
    cpu_backend.install(monkeypatch)
    criticalkv_backend.install(monkeypatch)
    model, ids = tiny_model("llama"), distinct_ids(120, seed=5)
    steps = [torch.tensor([[10 + t], [40 + t]]) for t in range(12)]

    def drive(cache, **fw):
        model.model(input_ids=ids, past_key_values=cache, **fw)
        for t, x in enumerate(steps):
            extra = {"cache_position": torch.tensor([ids.shape[1] + t])} if fw else {}
            model.model(input_ids=x, past_key_values=cache, **extra)

    def reference(kvpress):
        cache = DynamicCache()
        press = kvpress.PrefillDecodingPress(
            prefilling_press=kvpress.CriticalKVPress(kvpress.KnormPress(0.5)),
            decoding_press=kvpress.DecodingPress(kvpress.KnormPress(), compression_interval=5, target_size=64))
        with press(model):
            drive(cache, cache_position=torch.arange(ids.shape[1]))
        return {"len": cache.get_seq_length(), **{f"sig{i}": rows_signature(la.keys, la.values)
                                                   for i, la in enumerate(cache.layers)}}

    want = ref("prefill_decoding/critical_knorm", reference)
    cache = DynamicCache()
    press = PrefillDecodingPress(prefilling_press=CriticalKVPress(KnormPress(0.5)),
                                 decoding_press=DecodingPress(KnormPress(), compression_interval=5, target_size=64))
    with press(model):
        drive(cache)
    assert cache.get_seq_length() == int(want["len"])
    for i, la in enumerate(cache.layers):
        close(rows_signature(la.keys, la.values), want[f"sig{i}"], f"layer {i}")
