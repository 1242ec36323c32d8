"""CAMPress on the GPU-less box: the C ABI's checks of kvp_cam_compress, the workspace formula and launch count of scorer
id 17, the wrapper's argument list, the float64 definition of tests/cam_backend.py against the UNMODIFIED reference,
and the press on float32 tiny Llama and Qwen3 models with the float64 stand-ins in place of the kernels.

Statuses: every argument made invalid on its own (or set to another valid value), and every pair of such changes,
against a restatement of the documented check order (include/kvpress_b200.h). The pointers are fake and never
dereferenced: the calls run in a child process that sees no GPU, so a call that passes every check fails at its first
CUDA call with KVP_ERR_CUDA (-6).

Reference: what the reference's `CAMPress.compress` returns on seeded float32 inputs, and the caches its press leaves
on float32 tiny models, are stored in tests/golden/cam_reference.npz, with the reference's torch.bernoulli(p) replaced
by (u < p) on the uniforms this side draws too. To re-record it from a checkout of the reference (located as in
oracle/build_ref.py):
    KVP_RECORD_CAM=1 python -m pytest tests/test_cam_host.py
"""
import ctypes
import re
from pathlib import Path

import pytest
import torch
from transformers import DynamicCache

from kvpress_b200 import (CAMPress, KnormPress, KVPressTextGenerationPipeline, PrefillDecodingPress,
                          StreamingLLMPress, TOVAPress, native)
from kvpress_b200.presses import cam_press
from tests import abi_cases, cam_backend as CB, cpu_backend
from tests.abi_cases import GOOD, ODD16
from tests.support import TO_32BIT, close, rec, reference_store, rows_signature  # noqa: F401  (rec: fixture)
from tests.tiny_models import tiny_model, word_tokenizer, words

HEADER = Path(__file__).resolve().parent.parent / "include" / "kvpress_b200.h"
STORE = Path(__file__).resolve().parent / "golden" / "cam_reference.npz"
ODD4 = 0x10002  # 2-byte but not 4-byte aligned


# --------------------------------------------------------------------------------------------------
# C ABI statuses
# --------------------------------------------------------------------------------------------------
def _checks(f, a, compress):
    """operands null -> uniforms null with n_merge != 0 -> alignment -> merge_budget and n_merge."""
    if None in (a["scores"], a["sstride"], a["attn"], a["astride"], a["attn_out"], a["ostride"]):
        return -1
    if a["u"] is None and a["n_merge"] != 0:
        return -1
    if a["scores"] % 2 or any(x is not None and x % 4 for x in (a["attn"], a["attn_out"], a["u"], a["idx_out"],
                                                                  a["midx"], a["mprob"])):
        return -4
    if a["budget"] < 1 or not 0 <= a["n_merge"] <= f["S"] - f["n_kept"]:
        return -7
    return 0


ABI = abi_cases.Spec(
    scorer=native.SCORER_CAM,
    slots={"kvp_cam_compress": "scores sstride K V attn astride n_merge budget u K_out V_out attn_out ostride idx_out "
                                "midx mprob ws ws_bytes stream"},
    valid=dict(scores=GOOD, sstride="sstride", K=GOOD, V=GOOD, attn=GOOD, astride="sstride", n_merge=100, budget=32,
               u=GOOD, K_out=GOOD, V_out=GOOD, attn_out=GOOD, ostride="sstride", idx_out=GOOD, midx=GOOD, mprob=GOOD,
               ws=GOOD, ws_bytes="enough", stream=0),
    changes={
        "p": {"null": None},
        "dtype": {"1": 1, "3": 3},
        "S": {"0": 0, "1": 1},
        "D": {"8": 8, "12": 12, "264": 264},
        "n_kept": {"-1": -1, "0": 0, "900": 900, "1000": 1000},
        "v_stride": {"s100": (256000, 128000, 100)},
        "scores": {"null": None, "odd": GOOD + 1},
        "sstride": {"null": None},
        "K": {"null": None, "odd": ODD16},
        "V": {"null": None},
        "attn": {"null": None, "odd": ODD4},
        "astride": {"null": None},
        "n_merge": {"-1": -1, "0": 0, "500": 500, "501": 501},
        "budget": {"0": 0, "1": 1, "big": 1 << 30},
        "u": {"null": None, "odd": ODD4},
        "K_out": {"odd": ODD16},
        "V_out": {"null": None},
        "attn_out": {"null": None, "odd": ODD4},
        "ostride": {"null": None},
        "idx_out": {"null": None, "odd": ODD4},
        "midx": {"null": None, "odd": ODD4},
        "mprob": {"null": None, "odd": ODD4},
        "ws": {"null": None, "odd": ODD16},
        "ws_bytes": {"short": "short"},
    },
    operands={"compress": ([], [])},
    checks=_checks,
)


def test_every_status_of_kvp_cam_compress_follows_the_check_order():
    want = abi_cases.assert_statuses("tests.test_cam_host", 1000)
    assert want["kvp_cam_compress(valid)"] == -6
    assert want["kvp_cam_compress(n_merge=0,u=null)"] == -6  # no uniforms needed without candidates
    assert want["kvp_cam_compress(n_kept=0,K=null)"] == 0


def _problem(B=1, H=8, S=4096, D=128, n_kept=2048):
    p = native.KvpProblem()
    p.B, p.Hkv, p.Hq, p.S, p.D, p.n_kept, p.dtype = B, H, H, S, D, n_kept, 0
    for i, s in enumerate((H * S * D, S * D, D)):
        p.k_stride[i] = p.v_stride[i] = s
    return p


def _align(x):
    return (x + 255) // 256 * 256


def cam_bytes(B, H, S, n_kept):
    n_tiles = (S + 255) // 256
    sel = [B * 1024, B * 1024, (3 * B + 64) * 4, B * n_tiles * 8, B * n_tiles * 256 * 2, B * n_tiles * 264 * 2, B * 8]
    cam = [4 * B * n_kept, 4 * B * (S - n_kept), 4 * B * (S - n_kept), 4 * B * H * (S - n_kept)]
    return sum(_align(x) for x in sel + cam)


@pytest.mark.parametrize("B,H,S,n_kept", [(1, 8, 2560, 2048), (1, 8, 131584, 2048), (3, 2, 1000, 1), (2, 4, 7, 7)])
def test_workspace_formula(B, H, S, n_kept):
    assert native.workspace_bytes(_problem(B, H, S, 128, n_kept), native.SCORER_CAM) == cam_bytes(B, H, S, n_kept)


def test_workspace_monotone_in_S():
    sizes = [native.workspace_bytes(_problem(S=S, n_kept=100), native.SCORER_CAM) for S in range(100, 5000, 37)]
    assert sizes == sorted(sizes)


def test_ids_and_launch_count():
    lib = native.load()
    n = ctypes.c_int()
    assert lib.kvp_launches_per_compress(ctypes.byref(_problem()), 17, ctypes.byref(n)) == 0 and n.value == 6
    for unknown in (10, 12, 15):
        assert lib.kvp_launches_per_compress(ctypes.byref(_problem()), unknown, ctypes.byref(n)) == -7
    assert native.SCORER_CAM == 17


def test_wrapper_argument_list():
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    params = [a.strip() for a in re.search(r"kvp_status\s+kvp_cam_compress\(([^)]*)\)", text).group(1).split(",")]
    _, argtypes = native.SIGNATURES["kvp_cam_compress"]
    assert len(argtypes) == len(params)
    for t, decl in zip(argtypes, params):
        if "*" in decl or decl.startswith("kvp_stream_t"):
            assert t in (ctypes.c_void_p, native._PP, native._PI64), decl
        elif decl.startswith("size_t"):
            assert t is ctypes.c_size_t, decl
        else:
            assert t is ctypes.c_int32, decl


def test_wrapper_passes_its_arguments(rec):  # noqa: F811
    B, H, S, D, n_kept, n_merge = 2, 3, 50, 64, 20, 7
    keys, values = torch.randn(B, H, S, D).bfloat16(), torch.randn(B, H, S, D).bfloat16()
    scores = torch.randn(B, H, S).bfloat16()
    cap = torch.zeros(B, H, 80)
    out = torch.zeros(B, H, 64)
    u = torch.rand(B, H, n_merge)
    native.cam_compress(scores, keys, values, cap[..., :S], out[..., :n_kept], n_merge, 4, u, n_kept,
                        return_indices=True, return_plan=True)
    name, fields, args = rec.calls[-1]
    assert name == "kvp_cam_compress" and fields["n_kept"] == n_kept and fields["S"] == S
    assert list(args[1]) == [H * S, S] and list(args[5]) == [H * 80, 80] and list(args[12]) == [H * 64, 64]
    assert args[6:8] == [n_merge, 4]


# --------------------------------------------------------------------------------------------------
# the float64 definition against the unmodified reference
# --------------------------------------------------------------------------------------------------
ref = reference_store(STORE, "KVP_RECORD_CAM", TO_32BIT)


class _Uniforms:
    """One seeded stream of uniforms, drawn in the order the compactions ask for them."""

    def __init__(self, seed):
        self.g = torch.Generator().manual_seed(seed)

    def __call__(self, shape, device=None):
        return torch.rand(shape, generator=self.g)


def _bernoulli_from(draw):
    return lambda p, *a, **k: (draw(p.shape) < p).to(p.dtype)


class _Layer(torch.nn.Module):
    layer_idx = 0


# (name, S, n_kept, k, merge_budget, scores kind, running sum kind)
DEFINITION = [
    ("knorm", 60, 32, 16, 4, "knorm", "rand"),
    ("streaming", 60, 32, 16, 4, "streaming", "rand"),
    ("tova", 60, 32, 16, 4, "tova", "rand"),
    ("budget-1", 50, 20, 12, 1, "knorm", "rand"),
    ("budget-32", 90, 40, 30, 32, "knorm", "rand"),
    ("budget-above-n_kept", 50, 20, 12, 25, "knorm", "rand"),
    ("k-above-evicted", 40, 30, 25, 4, "knorm", "rand"),
    ("after-last-kept", 40, 20, 20, 4, "last", "rand"),
    ("zero-sum", 50, 24, 20, 4, "knorm", "zero"),
    ("zero-window", 50, 24, 20, 4, "streaming", "zero-window"),
]


def _definition_inputs(S, n_kept, kind, sum_kind, seed):
    g = torch.Generator().manual_seed(seed)
    keys, values = torch.randn(2, 2, S, 16, generator=g), torch.randn(2, 2, S, 16, generator=g)
    if kind == "knorm":
        scores = -keys.norm(dim=-1)
    elif kind == "streaming":
        scores = torch.ones(2, 2, S)
        scores[:, :, 4: 4 + S - n_kept] = 0
    elif kind == "tova":
        shared = torch.softmax(torch.randn(2, 1, S, generator=g), -1)
        scores = shared.expand(2, 2, S).clone()
    else:  # the best scores first: the candidates lie after the last kept row
        scores = torch.linspace(1, 0, S).expand(2, 2, S).clone()
    A = torch.rand(2, 2, S, generator=g)
    if sum_kind == "zero":
        A.zero_()
    elif sum_kind == "zero-window":
        A[:, :, S - (n_kept - 4):] = 0  # the kept recent rows hold nothing: a positive A[e] over a zero mean
    return keys, values, scores, A


@pytest.mark.parametrize("name,S,n_kept,k,budget,kind,sum_kind", DEFINITION, ids=[d[0] for d in DEFINITION])
def test_float64_definition_is_the_reference(monkeypatch, ref, name, S, n_kept, k, budget, kind, sum_kind):
    keys, values, scores, A = _definition_inputs(S, n_kept, kind, sum_kind, S + k)
    n_merge = min(k, S - n_kept)

    def reference(kvpress):
        from kvpress.presses.cam_press import CAMPress as RefCAM

        class Base(kvpress.ScorerPress):
            def score(self, *a, **kw):
                return scores.clone()

        press = RefCAM(base_press=Base(), target_size=n_kept, merge_budget=budget)
        press.layer_step_counts[0] = k
        press._running_attn_sum[0] = A.clone()
        with monkeypatch.context() as m:
            m.setattr(torch, "bernoulli", _bernoulli_from(_Uniforms(S)))
            kk, vv = press.compress(_Layer(), None, keys, values.clone(), A, {})
        return {"keys": kk, "values": vv, "attn": press._running_attn_sum[0]}

    want = ref(f"definition/{name}", reference)
    u = _Uniforms(S)((2, 2, n_merge))
    k_out, v64, a_out, kept, cand, p = CB.cam64(scores, keys, values, A, n_merge, budget, u, n_kept)
    close(k_out, want["keys"], name)
    close(v64.float(), want["values"], name)
    close(a_out.float(), want["attn"], name)
    if kind == "streaming":
        first_recent = S - (n_kept - 4)
        assert torch.equal(cand[0], torch.arange(first_recent - n_merge, first_recent))
    if name == "after-last-kept":
        assert (kept.max(-1).values.unsqueeze(-1) < cand).all()
    if sum_kind == "zero":
        assert (p == 0).all()
    if sum_kind == "zero-window":
        assert (p == 1).all()


# --------------------------------------------------------------------------------------------------
# the press on float32 tiny models
# --------------------------------------------------------------------------------------------------
PRESSES = {
    "knorm": lambda m: m.CAMPress(base_press=m.KnormPress(), compression_interval=3, target_size=24),
    "streaming": lambda m: m.CAMPress(base_press=m.StreamingLLMPress(), compression_interval=3, target_size=24),
    "tova": lambda m: m.CAMPress(base_press=m.TOVAPress(), compression_interval=3, target_size=24),
    "prefill_decoding": lambda m: m.PrefillDecodingPress(
        prefilling_press=m.KnormPress(compression_ratio=0.6),
        decoding_press=m.CAMPress(base_press=m.KnormPress(), compression_interval=3, target_size=24)),
}


class _Ours:
    CAMPress, KnormPress, StreamingLLMPress, TOVAPress, PrefillDecodingPress = (
        CAMPress, KnormPress, StreamingLLMPress, TOVAPress, PrefillDecodingPress)


def _decode(make, kvpress, family, record, monkeypatch):
    """A prefill of 40 tokens, then 14 decoding steps of fixed tokens through the press's hooks."""
    model = tiny_model(family)
    press = make(kvpress)
    ids = torch.arange(10, 50).unsqueeze(0)
    cache = DynamicCache()
    draw = _Uniforms(7)
    with monkeypatch.context() as m:
        if record:
            m.setattr(torch, "bernoulli", _bernoulli_from(draw))
        else:
            m.setattr(cam_press, "draw_uniforms", draw)
        with press(model):
            model.model(input_ids=ids, past_key_values=cache, cache_position=torch.arange(40))
            for step in range(14):
                model.model(input_ids=torch.tensor([[60 + step]]), past_key_values=cache,
                            cache_position=torch.tensor([40 + step]), position_ids=torch.tensor([[40 + step]]))
            cam = press.decoding_press if hasattr(press, "decoding_press") else press
            sums = {i: cam._running_attn_sum[i] for i in range(len(cache.layers))}  # reset when the call ends
    out = {"len": cache.get_seq_length()}
    for i, la in enumerate(cache.layers):
        out[f"keys{i}"], out[f"values{i}"] = la.keys, la.values
        out[f"attn{i}"] = sums[i] if torch.is_tensor(sums[i]) else sums[i].view()
    return out


@pytest.mark.parametrize("family", ["llama", "qwen3"])
@pytest.mark.parametrize("name", sorted(PRESSES))
def test_press_leaves_the_reference_cache(monkeypatch, ref, name, family):
    want = ref(f"press/{name}/{family}", lambda kvpress: _decode(PRESSES[name], kvpress, family, True, monkeypatch))
    cpu_backend.install(monkeypatch)
    CB.install(monkeypatch)
    got = _decode(PRESSES[name], _Ours, family, False, monkeypatch)
    assert got["len"] == int(want["len"])
    assert 24 <= got["len"] <= 24 + 3 - 1  # the reference's test_decoding_compression bounds
    for i in range(2):
        if name == "prefill_decoding":
            # the reference's prefill press leaves its rows in score order, and CaM's windows follow the cache order:
            # the kept keys are the same rows, the merges legitimately differ
            k_got, k_want = got[f"keys{i}"], torch.as_tensor(want[f"keys{i}"])
            close(rows_signature(k_got, 0 * k_got), rows_signature(k_want, 0 * k_want), f"{family} layer {i}")
            continue
        for part in ("keys", "values", "attn"):
            close(got[f"{part}{i}"], want[f"{part}{i}"], f"{name} {family} layer {i} {part}")


def test_pipeline_bounds_and_reset_between_calls(monkeypatch):
    cpu_backend.install(monkeypatch)
    CB.install(monkeypatch)
    pipe = KVPressTextGenerationPipeline(model=tiny_model(), tokenizer=word_tokenizer(), device="cpu")
    press = CAMPress(base_press=KnormPress(), compression_interval=4, target_size=32)
    for seed in (1, 2):
        cache = DynamicCache()
        pipe(words(70 + 10 * seed, seed=seed), question=words(5, seed=3), press=press, cache=cache, max_new_tokens=20)
        for la in cache.layers:
            assert 32 <= la.keys.shape[2] <= 32 + 4 - 1
        # the press's context manager resets its per-sequence state when the call ends
        assert press._running_attn_sum == {} and not press.layer_step_counts
    # prefill drops a layer's state inside one call, as the reference's hook does
    press._running_attn_sum[0] = object()
    press.layer_step_counts[0] = 5
    press._on_prefill(0)
    assert 0 not in press._running_attn_sum and press.layer_step_counts[0] == 0


def test_base_press_must_be_a_scorer_press():
    from kvpress_b200 import AdaKVPress, SnapKVPress

    with pytest.raises(TypeError, match="ScorerPress"):
        CAMPress(base_press=AdaKVPress(SnapKVPress()))
    with pytest.raises(AssertionError):
        CAMPress(base_press=KnormPress(), merge_budget=0)
    press = CAMPress(base_press=KnormPress())
    assert (press.compression_interval, press.target_size, press.hidden_states_buffer_size, press.merge_budget) == (
        512, 2048, 256, 32)
