"""kvp_think_prune on the H100 against the float64 definition (include/kvpress_b200.h, kvp_think_prune), from the same
16-bit inputs (tests/think_backend.py).

The bar, for every call:
  - scores: |score - score64| <= 2^-16 |score64| (the header's a-priori bound; NaN and inf where float64 has them);
  - selection: the pruned set is exactly the tie / NaN rule applied to the kernel's own fp32 scores, and it equals the
    float64 set unless the bound leaves the boundary undecided (a float64 gap at the boundary within 2^-15 relative);
  - zeroing: every element of a pruned channel is bit 0, every other element of K is bit-identical, V and the guard
    bands around the view are untouched.
"""
import ctypes
import re
from pathlib import Path

import pytest
import torch
from transformers import DynamicCache

from kvpress_b200 import (ComposedPress, KnormPress, KVPressTextGenerationPipeline, PrefillDecodingPress, SnapKVPress,
                          ThinKPress, native)
from tests import think_backend as TB
from tests.tiny_models import distinct_ids, tiny_llama, word_tokenizer, words

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF16, FP16 = torch.bfloat16, torch.float16
EPS = 2.0 ** -16
UNIT = 256
HEADER = Path(__file__).resolve().parent.parent / "include" / "kvpress_b200.h"


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def inputs(B, H, G, S, D, w, dtype, seed=0):
    g = _gen(seed)
    scale = torch.rand(D, generator=g, device=DEV) * 2 + 0.05
    k = (torch.randn(B, H, S, D, generator=g, device=DEV) * scale).to(dtype)
    q = (torch.randn(B, H * G, w, D, generator=g, device=DEV) * (0.5 + scale.flip(0))).to(dtype)
    return k, q


def bits(t):
    return t.view(torch.int16)


def check(k_before, k_after, q, n_pruned, pruned, scores, what=""):
    """The bar of the module docstring for one call on K (k_before: a copy of the input)."""
    B, H, S, D = k_before.shape
    s64 = TB.scores64(k_before, q)
    nan = s64.isnan()
    assert torch.equal(scores.isnan(), nan), what
    fin = s64.isfinite()
    assert torch.equal(scores.isinf() & ~nan, s64.isinf()), what
    err = (scores.double() - s64).abs()[fin]
    assert (err <= EPS * s64.abs()[fin]).all(), (what, float((err / s64.abs()[fin].clamp_min(1e-300)).max()))
    assert torch.equal(scores[s64.isinf()], s64[s64.isinf()].float()), what
    mask = TB.pruned_mask(scores, n_pruned)
    assert (mask.sum(-1) == n_pruned).all(), what
    want_idx = mask.nonzero()[:, 2].view(B, H, n_pruned)
    assert torch.equal(pruned.long(), want_idx), what
    m64 = TB.pruned_mask(s64, n_pruned)
    differ = (mask != m64).any(-1)
    if differ.any() and 0 < n_pruned < D:
        kept_min = s64.masked_fill(m64, float("inf")).amin(-1)
        pruned_max = s64.masked_fill(~m64, float("-inf")).amax(-1)
        gap = (kept_min - pruned_max)[differ]
        assert (gap <= 2 * EPS * kept_min[differ].abs()).all(), (what, gap)
    m = mask.unsqueeze(2).expand_as(k_after)
    assert (bits(k_after)[m] == 0).all(), what
    assert torch.equal(bits(k_after)[~m], bits(k_before)[~m]), what


def run(k, q, n_pruned, what=""):
    before = k.clone()
    out, pruned, scores = native.think_prune(k, q, n_pruned, return_pruned=True, return_scores=True)
    torch.cuda.synchronize()
    assert out is k
    if n_pruned == 0:
        assert pruned is None and scores is None and torch.equal(bits(k), bits(before))
        return None
    check(before, k, q, n_pruned, pruned, scores, what)
    return pruned, scores


# --------------------------------------------------------------------------------------------------
# instantiations
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", list(range(8, 257, 8)))
@pytest.mark.parametrize("dtype", [BF16, FP16], ids=["bf16", "fp16"])
def test_instantiations(dtype, D):
    """Every head_dim, both dtypes, G in {1, 2, 4, 8} and window in {1, 32, 257}."""
    for G in (1, 2, 4, 8):
        for w in (1, 32, 257):
            k, q = inputs(2, 2, G, 300, D, w, dtype, seed=D * 10 + G + w)
            run(k, q, D // 2, f"G{G} w{w}")


@pytest.mark.parametrize("S", [1, UNIT - 1, UNIT, UNIT + 1, 4099, 32768, 131072])
def test_sizes(S):
    """n_pruned 0, 1, D/2, D-1 and D at S around one unit and up to 128k."""
    D = 128
    for n in (0, 1, D // 2, D - 1, D):
        k, q = inputs(1, 2, 4, S, D, 32, BF16, seed=S + n)
        run(k, q, n, f"S{S} n{n}")


def test_3000_rows():
    k, q = inputs(3, 1000, 1, 70, 64, 4, FP16, seed=7)
    run(k, q, 20)


# --------------------------------------------------------------------------------------------------
# planted values
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [BF16, FP16], ids=["bf16", "fp16"])
def test_planted_ties_nan_inf_and_zero_channels(dtype):
    """Exact ties keep the lower channel; NaN is pruned last, NaNs by channel; inf, and inf * 0 = NaN; all-zero channels
    score 0. The rules hold exactly at every n_pruned."""
    B, H, G, S, D, w = 1, 4, 2, 600, 32, 8
    k, q = inputs(B, H, G, S, D, w, dtype, seed=3)
    # head 0: channels 3, 9, 20 are copies of channel 5 (exact ties), channel 7 is zero
    for c in (3, 9, 20):
        k[0, 0, :, c] = k[0, 0, :, 5]
    q[0, 0:2, :, [3, 9, 20]] = q[0, 0:2, :, 5:6]
    k[0, 0, :, 7] = 0
    # head 1: NaN keys in channels 4 and 11, an inf key in channel 6
    k[0, 1, 17, 4] = float("nan")
    k[0, 1, 300, 11] = float("nan")
    k[0, 1, 5, 6] = float("inf")
    # head 2: an inf key in channel 2 whose queries are 0 (inf * 0 = NaN), zero queries in channel 8
    k[0, 2, 9, 2] = float("-inf")
    q[0, 4:6, :, 2] = 0
    q[0, 4:6, :, 8] = 0
    # head 3: every channel ties
    k[0, 3] = 1
    q[0, 6:8] = 1
    for n in range(D + 1):
        kk = k.clone()
        r = run(kk, q, n, f"n{n}")
        if r is None:
            continue
        pruned, scores = r
        # check() holds the pruned sets to the tie and NaN rules exactly; here the planted scores themselves
        assert pruned[0, 3].tolist() == list(range(D - n, D))  # all tied: the highest channels go first
        assert torch.equal(scores[0, 0, [3, 9, 20]], scores[0, 0, 5].expand(3)) and scores[0, 0, 7] == 0
        assert scores[0, 1, 4].isnan() and scores[0, 1, 11].isnan() and scores[0, 1, 6].isinf()
        assert scores[0, 2, 2].isnan() and scores[0, 2, 8] == 0
        nan1 = [c for c in pruned[0, 1].tolist() if c in (4, 11)]
        assert nan1 == ([4, 11] if n == D else [11] if n == D - 1 else [])  # NaN last, the higher channel first


# --------------------------------------------------------------------------------------------------
# layouts, guard bands, determinism
# --------------------------------------------------------------------------------------------------
def test_strided_views_guards_and_values_untouched():
    """A slice of a longer cache and permuted batch / head strides: only the view's pruned channels change; the rows
    outside the slice, the values interleaved with the keys and the guard bands are bit-identical."""
    B, H, G, S, D, w = 2, 3, 4, 1000, 64, 16
    g = _gen(11)
    store = torch.randn(H, B, 2, S + 40, D, generator=g, device=DEV).to(BF16)  # [h][b][k / v][position][channel]
    guard = torch.randn(4096, generator=g, device=DEV).to(BF16)
    arena = torch.cat([guard, store.flatten(), guard])
    before = arena.clone()
    view = arena[4096:4096 + store.numel()].view(H, B, 2, S + 40, D)
    k = view[:, :, 0, 20:20 + S].permute(1, 0, 2, 3)  # [B, H, S, D], permuted batch / head strides
    v = view[:, :, 1, 20:20 + S].permute(1, 0, 2, 3)
    q = torch.randn(B, H * G, w, D, generator=g, device=DEV).to(BF16)
    k_before, v_before = k.clone(), v.clone()
    _, pruned, scores = native.think_prune(k, q, 24, return_pruned=True, return_scores=True)
    torch.cuda.synchronize()
    check(k_before, k, q, 24, pruned, scores, "strided")
    assert torch.equal(bits(v), bits(v_before))
    touched = torch.zeros_like(arena, dtype=torch.bool)
    touched[4096:4096 + store.numel()].view(H, B, 2, S + 40, D)[:, :, 0, 20:20 + S] = True
    assert torch.equal(bits(arena)[~touched], bits(before)[~touched])


def test_determinism_batch_independence_and_schedules():
    """Two calls give bitwise-equal results; a row's results are the same alone and inside a batch, and at shapes that
    give one unit or many units per SM."""
    B, H, G, D, w = 4, 8, 4, 128, 32
    for S in (300, 40000):
        k, q = inputs(B, H, G, S, D, w, BF16, seed=S)
        a, b = k.clone(), k.clone()
        ra = native.think_prune(a, q, 64, True, True)
        rb = native.think_prune(b, q, 64, True, True)
        torch.cuda.synchronize()
        assert torch.equal(bits(a), bits(b)) and torch.equal(ra[1], rb[1]) and torch.equal(ra[2].view(torch.int32),
                                                                                         rb[2].view(torch.int32))
        for bi, hi in ((0, 0), (3, 5), (2, 7)):
            one = k[bi:bi + 1, hi:hi + 1].clone()
            r1 = native.think_prune(one, q[bi:bi + 1, hi * G:(hi + 1) * G].contiguous(), 64, True, True)
            torch.cuda.synchronize()
            assert torch.equal(r1[2][0, 0].view(torch.int32), ra[2][bi, hi].view(torch.int32))
            assert torch.equal(r1[1][0, 0], ra[1][bi, hi]) and torch.equal(bits(one[0, 0]), bits(a[bi, hi]))


def test_graph_capture_replay_and_no_allocation():
    k, q = inputs(1, 8, 4, 5000, 128, 32, BF16, seed=5)
    src = k.clone()
    pruned = torch.empty(1, 8, 64, dtype=torch.int32, device=DEV)
    lib = native.load()
    p = native.make_problem(k, k, k.shape[2], q.shape[1])
    ws = native._workspace(p, native.SCORER_THINK, k.device)

    call_p = lambda: native._check(lib.kvp_think_prune(ctypes.byref(p), k.data_ptr(), q.data_ptr(), 32, 64,  # noqa
                                                       pruned.data_ptr(), None, ws.data_ptr(), ws.numel(),
                                                       native._stream()), "kvp_think_prune")
    call_p()
    torch.cuda.synchronize()
    want_k, want_p = k.clone(), pruned.clone()
    used = torch.cuda.memory_allocated()
    k.copy_(src)
    call_p()
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == used
    assert torch.equal(bits(k), bits(want_k)) and torch.equal(pruned, want_p)
    k.copy_(src)
    pruned.zero_()
    graph = native.capture(call_p)
    for _ in range(2):
        k.copy_(src)
        pruned.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(bits(k), bits(want_k)) and torch.equal(pruned, want_p)


# --------------------------------------------------------------------------------------------------
# inputs past 2 GiB and 4 GiB
# --------------------------------------------------------------------------------------------------
TWO31, TWO32 = 1 << 31, 1 << 32
FAR_CASES = {"kvp_think_prune"}


def test_far_inputs_past_2_and_4_gib():
    """K, q_window, the outputs and the workspace of one arena, past the 2 GiB and 4 GiB offsets."""
    free, _ = torch.cuda.mem_get_info()
    if free < TWO32 + (1 << 28):
        pytest.skip("needs 4.3 GB of device memory")
    B, H, G, S, D, w = 1, 4, 4, 3000, 128, 32
    k0, q0 = inputs(B, H, G, S, D, w, BF16, seed=9)
    arena = torch.zeros(TWO32 + (1 << 26), dtype=torch.uint8, device=DEV)
    k_off, q_off = TWO32 + 4096, TWO31 + 8192
    k = arena[k_off:k_off + k0.numel() * 2].view(BF16).view(k0.shape)
    q = arena[q_off:q_off + q0.numel() * 2].view(BF16).view(q0.shape)
    k.copy_(k0)
    q.copy_(q0)
    p = native.make_problem(k, k, S, H * G)
    need = native.workspace_bytes(p, native.SCORER_THINK)
    ws_off = TWO32 + (1 << 25)
    out_off = TWO31 + (1 << 20)
    pruned = arena[out_off:out_off + B * H * 64 * 4].view(torch.int32).view(B, H, 64)
    scores = arena[out_off + 65536:out_off + 65536 + B * H * D * 4].view(torch.float32).view(B, H, D)
    lib = native.load()
    rc = lib.kvp_think_prune(ctypes.byref(p), k.data_ptr(), q.data_ptr(), w, 64, pruned.data_ptr(), scores.data_ptr(),
                             arena.data_ptr() + ws_off, need, native._stream())
    torch.cuda.synchronize()
    assert rc == 0
    check(k0, k, q0, 64, pruned, scores, "far")
    del arena


def test_every_think_entry_point_has_a_far_input_case():
    declared = set(re.findall(r"^(?:int|kvp_status) (kvp_think_\w+)\(", HEADER.read_text(), re.M))
    assert declared and declared <= FAR_CASES


# --------------------------------------------------------------------------------------------------
# the press on a tiny GPU Llama
# --------------------------------------------------------------------------------------------------
PRESSES = {
    "alone": lambda: ThinKPress(key_channel_compression_ratio=0.5, window_size=16),
    "snapkv-think": lambda: ComposedPress([SnapKVPress(0.5, window_size=16), ThinKPress(0.5)]),
    "think-knorm": lambda: ComposedPress([ThinKPress(0.5), KnormPress(0.5)]),
    "prefill_decoding": lambda: PrefillDecodingPress(prefilling_press=ThinKPress(0.75, window_size=8)),
}


def _prefill(model, ids, press):
    cache = DynamicCache()
    seen = []
    real = native.think_prune

    def spy(keys, *a, **kw):
        seen.append(keys)
        return real(keys, *a, **kw)

    native.think_prune = spy
    try:
        with press(model):
            model.model(input_ids=ids, past_key_values=cache)
    finally:
        native.think_prune = real
    torch.cuda.synchronize()
    return cache, seen


@pytest.mark.parametrize("name", sorted(PRESSES))
def test_press_on_a_tiny_llama(monkeypatch, name):
    """The kernel against the float64 stand-in in the same forward: the same cache, bit for bit, and the pruned keys
    are the cache's own tensors."""
    model = tiny_llama(dtype=BF16, device=DEV, head_dim=64)
    ids = distinct_ids(200, seed=4, device=DEV)
    with torch.no_grad():
        got, seen = _prefill(model, ids, PRESSES[name]())
        assert len(seen) == 2
        if name != "think-knorm":  # there Knorm replaces the pruned tensors by its compacted ones
            assert all(any(s is la.keys for la in got.layers) for s in seen)
        monkeypatch.setattr(native, "think_prune", TB.think_prune64)
        want, _ = _prefill(model, ids, PRESSES[name]())
    for a, b in zip(got.layers, want.layers):
        assert torch.equal((a.keys == 0).all(dim=2), (b.keys == 0).all(dim=2))
        assert torch.equal(bits(a.keys), bits(b.keys)) and torch.equal(bits(a.values), bits(b.values))


def test_pipeline_generates_with_think():
    model = tiny_llama(dtype=BF16, device=DEV, head_dim=64)
    pipe = KVPressTextGenerationPipeline(model=model, tokenizer=word_tokenizer(), device=DEV)
    out = pipe(words(300, seed=1), question=words(5, seed=2), press=ComposedPress([SnapKVPress(0.5, window_size=16), ThinKPress(0.5)]),
               max_new_tokens=4)
    assert isinstance(out["answer"], str)
