"""KVzapPress / DMSPress without a GPU: the C ABI's statuses, workspace formula and launch count, the wrapper argument
lists, the float64 definitions of tests/kvzap_backend.py against torch and against the UNMODIFIED reference, the presses
on float32 tiny Llama and Qwen3 models (prefill and decoding steps, float64 stand-ins in place of the kernels) against
the masks and ratios the reference's presses leave, checkpoint loading and the press errors.

The reference results are stored in tests/golden/kvzap_reference.npz; to re-record them from a checkout of the
reference (located as in oracle/build_ref.py):
    KVP_RECORD_KVZAP=1 python -m pytest tests/test_kvzap_host.py
"""
import ctypes
import math

import pytest
import torch

from tests import abi_cases, cpu_backend, kvzap_backend as KB

GOOD = abi_cases.GOOD


def _statuses():
    """(name, status) of representative calls through the C ABI, each breaking one check of the documented order."""
    nat, lib = abi_cases.load_native()
    xs = (ctypes.c_int64 * 2)(1000 * 4096, 4096)
    ss = (ctypes.c_int64 * 2)(2000, 1000)
    out = []

    def score(name, hidden=4096, hd=512, x=GOOD, w1=GOOD, b1=GOOD, w2=GOOD, b2=GOOD, stride=xs, scores=GOOD,
              ws=GOOD, ws_bytes=1 << 40, **fields):
        p = abi_cases.problem(nat, fields, abi_cases.FIELDS)
        out.append((name, lib.kvp_kvzap_score(ctypes.byref(p), x, stride, hidden, hd, w1, b1, w2, b2, scores, ws,
                                              ws_bytes, None)))

    score("valid")
    score("dtype", dtype=5)
    score("scores null", scores=None)
    score("scores odd", scores=GOOD + 1)
    score("x null", x=None)
    score("w2 null", w2=None)
    score("w2 null linear", w2=None, b2=None, hd=0)
    score("x unaligned", x=abi_cases.ODD16)
    score("b2 odd", b2=GOOD + 1)
    score("hidden 0", hidden=0)
    score("stride odd", stride=(ctypes.c_int64 * 2)(1000 * 4096, 4095))
    score("stride short", stride=(ctypes.c_int64 * 2)(1000 * 4096, 4088))
    score("hidden 4100", hidden=4100, stride=(ctypes.c_int64 * 2)(1000 * 4104, 4104))
    score("hidden 16392", hidden=16392, stride=(ctypes.c_int64 * 2)(1000 * 16392, 16392))
    score("hd 2056", hd=2056)
    score("Hkv 33", Hkv=33, Hq=33)
    score("ws null", ws=None)
    score("ws odd", ws=abi_cases.ODD16)
    score("ws small", ws_bytes=16)

    def evict(name, dtype=0, B=2, H=1, n=1000, n_evict=10, scores=GOOD, count=GOOD, ws=GOOD, ws_bytes=256):
        out.append((name, lib.kvp_threshold_evict(dtype, B, H, n, scores, ss, n_evict, ctypes.c_float(0.5), 3, GOOD,
                                                  GOOD, GOOD, count, ws, ws_bytes, None)))

    evict("evict valid")
    evict("evict dtype", dtype=2)
    evict("evict n 0", n=0)
    evict("evict n_evict", n_evict=1001)
    evict("evict scores null", scores=None)
    evict("evict count odd", count=GOOD + 4)
    evict("evict ws small", ws_bytes=256, B=64, H=1)
    evict("evict ws per tile", ws_bytes=256, B=32, H=1, n=4097, n_evict=1)
    evict("evict grid", B=1 << 20, H=32, n=1 << 20, n_evict=1)
    sizes = []
    for B, H, S in [(1, 8, 1), (1, 8, 32), (2, 8, 17), (1, 8, 33), (2, 4, 1000)]:
        p = abi_cases.problem(nat, dict(B=B, Hkv=H, Hq=H, S=S, n_kept=min(S, 1)), abi_cases.FIELDS)
        n = ctypes.c_size_t(0)
        lib.kvp_workspace_bytes(ctypes.byref(p), nat.SCORER_KVZAP, ctypes.byref(n))
        g = ctypes.c_size_t(0)
        lib.kvp_workspace_bytes(ctypes.byref(p), nat.SCORER_GENERIC, ctypes.byref(g))
        c = ctypes.c_int(0)
        lib.kvp_launches_per_compress(ctypes.byref(p), nat.SCORER_KVZAP, ctypes.byref(c))
        sizes.append((B, H, S, n.value, g.value, c.value))
    return out, sizes


@pytest.fixture(scope="module")
def abi():
    return abi_cases.in_child("tests.test_kvzap_host:_statuses")


EXPECTED = {
    "valid": -6, "dtype": -3, "scores null": -1, "scores odd": -4, "x null": -1, "w2 null": -1, "w2 null linear": -6,
    "x unaligned": -4, "b2 odd": -4, "hidden 0": -7, "stride odd": -4, "stride short": -4, "hidden 4100": -2,
    "hidden 16392": -2, "hd 2056": -2, "Hkv 33": -2, "ws null": -1, "ws odd": -4, "ws small": -5,
    "evict valid": -6, "evict dtype": -3, "evict n 0": -2, "evict n_evict": -7, "evict scores null": -1,
    "evict count odd": -4, "evict ws small": -5, "evict ws per tile": -5, "evict grid": -2,
}


def test_statuses_follow_the_documented_check_order(abi):
    assert dict(abi[0]) == EXPECTED


def test_workspace_formula_and_launch_count(abi):
    for B, H, S, n, generic, launches in abi[1]:
        parts = 256 if B * S <= 32 else 16
        align = lambda v: (v + 255) // 256 * 256  # noqa: E731
        assert n == generic + align(4 * parts * H * B * S) + align(2 * B * H * S)
        assert launches == 5


def test_wrapper_argument_lists():
    from kvpress_b200 import native

    assert len(native.SIGNATURES["kvp_kvzap_score"][1]) == 13
    assert len(native.SIGNATURES["kvp_kvzap_compress"][1]) == 18
    assert len(native.SIGNATURES["kvp_threshold_evict"][1]) == 16
    assert native.SCORER_KVZAP == 18
    assert native.kvzap_supported(4096, 512, 8) and native.kvzap_supported(4096, 0, 32)
    assert not native.kvzap_supported(4100, 512, 8) and not native.kvzap_supported(4096, 2056, 8)
    assert not native.kvzap_supported(4096, 512, 33) and not native.kvzap_supported(16392, 0, 8)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("hd", [0, 64, 200])
def test_float64_definition_and_bound_hold_for_an_fp32_evaluation(dtype, hd):
    """An fp32 evaluation rounded once (what the kernels compute, in another order) lies inside the bound, and the
    float64 definition is the reference's nn modules evaluated in float64."""
    from kvpress_b200.presses.kvzap_press import KVzapConfig, KVzapModel, layer_weights

    torch.manual_seed(hd)
    m = KVzapModel(KVzapConfig(input_dim=512, output_dim=4, hidden_dim=hd or None, n_modules=1)).to(dtype)
    ws = tuple(None if w is None else w.detach().clone() for w in layer_weights(m.layers[0]))
    x = torch.randn(2, 77, 512).to(dtype)
    s64, E = KB.kvzap64(x, *ws)
    with torch.no_grad():
        ref = m.double()(x.double().reshape(-1, 1, 512))[:, 0].view(2, 77, 4).transpose(1, 2)
        assert torch.allclose(ref, s64, rtol=1e-12, atol=1e-12)
        w32 = [None if w is None else w.float() for w in ws]
        h = x.float() @ w32[0].t() + w32[1]
        if hd:
            h = torch.nn.functional.gelu(h) @ w32[2].t() + w32[3]
    assert KB.within_bound(h.transpose(1, 2).to(dtype), s64, E).all()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_threshold_is_rounded_to_the_score_dtype(dtype):
    s = torch.tensor([[[0.099609375, 0.0999755859375, float("nan"), -0.0, 0.0]]]).to(dtype)
    b, h, pos = KB.threshold_evict64(s, 5, 0.0998, 0)
    thr = torch.tensor(0.0998, dtype=torch.float32).to(dtype).double()
    want = [i for i, v in enumerate(s[0, 0].double().tolist()) if v < thr]
    assert pos.tolist() == want and not math.isnan(thr)


def test_model_loads_a_checkpoint_in_the_published_format(tmp_path):
    from kvpress_b200 import KVzapConfig, KVzapModel

    for hidden_dim, keys in [(None, {"layers.0.weight", "layers.0.bias", "layers.1.weight", "layers.1.bias"}),
                             (32, {f"layers.{i}.{j}.{w}" for i in (0, 1) for j in (0, 2) for w in ("weight", "bias")})]:
        m = KVzapModel(KVzapConfig(input_dim=64, output_dim=2, hidden_dim=hidden_dim, n_modules=2))
        assert set(m.state_dict()) == keys
        m.save_pretrained(tmp_path / str(hidden_dim))
        back = KVzapModel.from_pretrained(tmp_path / str(hidden_dim))
        assert back.config.hidden_dim == hidden_dim and back.config.n_modules == 2
        assert all(torch.equal(a, b) for a, b in zip(m.state_dict().values(), back.state_dict().values()))
        x = torch.randn(3, 2, 64)
        assert back(x).shape == (3, 2, 2)


def test_press_fields_and_errors():
    from kvpress_b200 import DMSPress, KnormPress, KVzapPress

    p = KVzapPress()
    assert p.model_type == "mlp" and p.kvzap_model_name is None and p.kvzap_model is None
    d = DMSPress(p)
    assert d.threshold is None and d.sliding_window_size == 128 and d.decoding is False
    with pytest.raises(AttributeError):
        d.compression_ratio = 0.5
    with pytest.raises(AssertionError):
        d.compression_ratio
    with pytest.raises(AssertionError):
        DMSPress(object())
    with pytest.raises(RuntimeError):
        p.weights(0, torch.empty(1))
    assert DMSPress(KnormPress(), threshold=1.0).threshold == 1.0


# --------------------------------------------------------------------------------------------------
# the float64 definitions and the presses against the unmodified reference
# --------------------------------------------------------------------------------------------------
from pathlib import Path  # noqa: E402

from transformers import DynamicCache  # noqa: E402

from tests.support import TO_32BIT, close, reference_store  # noqa: E402
from tests.tiny_models import tiny_model  # noqa: E402

STORE = Path(__file__).resolve().parent / "golden" / "kvzap_reference.npz"
ref = reference_store(STORE, "KVP_RECORD_KVZAP", TO_32BIT)


def _surrogate_state(kvpress_module, hidden, heads, hd, layers, seed):
    """A seeded surrogate model of `kvpress_module` (the reference's or ours) and its state dict."""
    torch.manual_seed(seed)
    m = kvpress_module.KVzapModel(kvpress_module.KVzapConfig(input_dim=hidden, output_dim=heads, hidden_dim=hd,
                                                             n_modules=layers))
    with torch.no_grad():  # biases large enough to matter, so a dropped bias fails
        for name, p in m.named_parameters():
            if name.endswith("bias"):
                p.normal_(0.0, 0.5)
    return m


class _Layer(torch.nn.Module):
    layer_idx = 1


@pytest.mark.parametrize("hd", [None, 32])
def test_float64_score_is_the_reference(ref, hd):
    def reference(kvpress):
        from kvpress.presses import kvzap_press as R

        m = _surrogate_state(R, 64, 2, hd, 2, 11)
        press = R.KVzapPress(model_type="mlp" if hd else "linear")
        press.kvzap_model = m
        x = torch.randn(2, 37, 64, generator=torch.Generator().manual_seed(5))
        scores = press.score(_Layer(), x, torch.zeros(2, 2, 37, 16), torch.zeros(2, 2, 37, 16), None, {})
        return {"x": x, "scores": scores, **{f"w.{k}": v for k, v in m.state_dict().items()}}

    want = ref(f"score/{'mlp' if hd else 'linear'}", reference)
    from kvpress_b200 import KVzapConfig, KVzapModel
    from kvpress_b200.presses.kvzap_press import layer_weights

    m = KVzapModel(KVzapConfig(input_dim=64, output_dim=2, hidden_dim=hd, n_modules=2))
    m.load_state_dict({k[2:]: torch.as_tensor(v) for k, v in want.items() if k.startswith("w.")})
    s64, _ = KB.kvzap64(torch.as_tensor(want["x"]), *layer_weights(m.layers[1]))
    close(s64, want["scores"], "score")


def _press(kvpress, kind, family, decoding):
    """DMSPress over KVzap (linear / MLP, seeded) or Knorm, with thresholds that evict some positions, not all."""
    if kind == "knorm":
        # Qwen3's normalised keys have norms within 1e-4 of 4
        threshold = -0.62 if family == "llama" else -3.99992
        return kvpress.DMSPress(kvpress.KnormPress(), threshold=threshold, sliding_window_size=8, decoding=decoding)
    hd = 32 if kind == "mlp" else None
    if hasattr(kvpress, "KVzapModel"):
        module = kvpress
    else:
        from kvpress.presses import kvzap_press as module
    m = _surrogate_state(module, 64, 2, hd, 2, 11 if family == "llama" else 12)
    press = kvpress.KVzapPress(model_type=kind)
    press.kvzap_model = m
    if not hasattr(kvpress, "KVzapModel"):  # the reference loads from the Hub unless told otherwise
        press.post_init_from_model = lambda model: None
    return kvpress.DMSPress(press, threshold=0.0, sliding_window_size=8, decoding=decoding)


def _run(kvpress, kind, family, decoding):
    """A prefill of 40 tokens, then 14 decoding steps of fixed tokens through the press's hooks."""
    model = tiny_model(family)
    press = _press(kvpress, kind, family, decoding)
    cache = DynamicCache()
    with torch.no_grad(), press(model):
        model.model(input_ids=torch.arange(10, 50).unsqueeze(0), past_key_values=cache,
                    cache_position=torch.arange(40))
        for step in range(14):
            model.model(input_ids=torch.tensor([[60 + step]]), past_key_values=cache,
                        cache_position=torch.tensor([40 + step]), position_ids=torch.tensor([[40 + step]]))
    out = {"ratio": torch.tensor([press.compression_ratios[i] for i in range(2)], dtype=torch.float64)}
    for i, layer in enumerate(model.model.layers):
        masked = layer.self_attn.masked_key_indices
        out[f"masked{i}"] = (torch.stack([torch.as_tensor(t) for t in masked]) if masked is not None
                             else torch.zeros(3, 0, dtype=torch.int64))
    return out


class _Ours:
    from kvpress_b200 import DMSPress, KnormPress, KVzapConfig, KVzapModel, KVzapPress  # noqa: F401


@pytest.mark.parametrize("decoding", [False, True])
@pytest.mark.parametrize("family", ["llama", "qwen3"])
@pytest.mark.parametrize("kind", ["linear", "mlp", "knorm"])
def test_dms_press_masks_what_the_reference_masks(monkeypatch, ref, kind, family, decoding):
    want = ref(f"dms/{kind}/{family}/{decoding}", lambda kvpress: _run(kvpress, kind, family, decoding))
    cpu_backend.install(monkeypatch)
    KB.install(monkeypatch)
    got = _run(_Ours, kind, family, decoding)
    close(got["ratio"], want["ratio"], "ratios")
    assert 0 < float(got["ratio"].min()) and float(got["ratio"].max()) < 1
    for i in range(2):
        assert torch.equal(got[f"masked{i}"], torch.as_tensor(want[f"masked{i}"]).long()), (kind, family, i)


def test_surrogate_is_reloaded_when_the_model_name_changes(monkeypatch):
    from types import SimpleNamespace

    from kvpress_b200 import KVzapPress
    from kvpress_b200.presses import kvzap_press

    loads = []
    monkeypatch.setattr(kvzap_press.KVzapModel, "from_pretrained",
                        classmethod(lambda cls, name: loads.append(name) or object()))
    model = lambda n: SimpleNamespace(config=SimpleNamespace(name_or_path=n))  # noqa: E731
    p = KVzapPress(model_type="linear")
    p.post_init_from_model(model("org/A"))
    p.post_init_from_model(model("org/A"))
    p.post_init_from_model(model("x/B"))
    assert loads == ["nvidia/KVzap-linear-A", "nvidia/KVzap-linear-B"] and p.kvzap_model_name.endswith("-B")
    own = object()
    q = KVzapPress(kvzap_model=own)
    q.post_init_from_model(model("org/A"))
    assert q.kvzap_model is own and len(loads) == 2
