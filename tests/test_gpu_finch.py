"""kvp_finch_* and kvp_scores_compress_chunked on the H100 against the float64 definition (include/kvpress_b200.h).

The bar:
  - scores: every context score within 1 ulp of the cache dtype of the float64 value. The kernel's fp32 evaluation
    (MUFU exp2 at 2 ulp, fp32 sums over at most G w S terms in a fixed order, one division) stays within a few
    2^-20 relative of the definition at these sizes, far below half an ulp of bf16 (2^-9) or fp16 (2^-12), so one
    rounding lands on one of the two dtype values around the float64 score. The window holds max + 1 rounded.
  - selection: exactly the per-chunk top-k of the kernel's own scores (window forced, ties to the lowest position),
    in ascending position order; K' and V' exact gathers, or K' re-rotated by (j - s) inv_freq (one of the admissible
    roundings of tests/gpu_support.py).
"""
import ctypes
import math

import pytest
import torch

from kvpress_b200 import FinchPress, KVPressTextGenerationPipeline, finch_wide_head, native
from tests.gpu_support import _gather, _same, assert_scores, rerotation_admissible, rope_inv_freq, tiny_gpu_llama
from tests.tiny_models import word_tokenizer, words

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF16, FP16 = torch.bfloat16, torch.float16


def inputs(B, H, G, S, D, w, dtype, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    k = torch.randn(B, H, S, D, generator=g, device=DEV).to(dtype)
    q = (torch.randn(B, H * G, w, D, generator=g, device=DEV) * 1.5).to(dtype)
    v = torch.randn(B, H, S, D, generator=g, device=DEV).to(dtype)
    return k, v, q


def chunked_topk(scores, w, L, ratio):
    """[B, H, n_kept] positions: per chunk the best max(1, int(len (1 - r))) (L = 0: the whole row, int(S (1 - r))),
    window forced, ties to the lowest position, ascending."""
    B, H, S = scores.shape
    s = scores.float().clone()
    s[..., S - w:] = float("inf")
    out = []
    bounds = [(0, S)] if not L else [(c, min(S, c + L)) for c in range(0, S, L)]
    for lo, hi in bounds:
        n = int(S * (1 - ratio)) if not L else max(1, int((hi - lo) * (1 - ratio)))
        order = torch.sort(-s[..., lo:hi], dim=-1, stable=True).indices[..., :n]
        out.append(torch.sort(order, dim=-1).values + lo)
    return torch.cat(out, dim=-1)


@pytest.mark.parametrize("dtype", [BF16, FP16])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("G", [1, 2, 3, 4, 8])
def test_scores_every_instantiation(dtype, D, G):
    for S, w in [(300, 1), (257, 64), (1000, 63), (1100, 65), (2048, 257)]:
        for normalize in (True, False):
            k, _, q = inputs(1, 2, G, S, D, w, dtype, seed=S + w)
            got = native.finch_score(k, q, w, normalize)
            assert_scores(got, k, q, w, normalize, f"{dtype} D{D} G{G} S{S} w{w} n{normalize}")


@pytest.mark.parametrize("normalize", [True, False])
@pytest.mark.parametrize("S,w", [(2, 1), (129, 128), (4096, 1024), (8192, 4095), (32768, 64), (131072, 1)])
def test_scores_windows_and_lengths(S, w, normalize):
    k, _, q = inputs(1, 2, 4, S, 128, w, BF16, seed=7)
    got = native.finch_score(k, q, w, normalize)
    assert_scores(got, k, q, w, normalize, f"S{S} w{w} n{normalize}")
    again = native.finch_score(k, q, w, normalize)
    assert torch.equal(got, again), "two calls differ"


@pytest.mark.parametrize("L", [0, 5, 127, 1024, 1025, 4096, 3000])
@pytest.mark.parametrize("rerotate", [False, True])
def test_compress_chunked_selection(L, rerotate):
    S, w, r = 3001, 40, 0.5
    k, v, q = inputs(2, 2, 4, S, 128, w, BF16, seed=L)
    inv = rope_inv_freq("theta10000", 128) if rerotate else None
    k_out, v_out, idx, scores = native.finch_compress(k, v, q, w, r, L or None, True, inv, True, True)
    want = chunked_topk(scores, w, L, r)
    assert torch.equal(idx.long(), want), f"L{L}: not the per-chunk top-k"
    assert _same(v_out, _gather(v, idx)), "V' is not an exact gather"
    if rerotate:
        adm = rerotation_admissible(k, idx, inv).view(torch.int16)
        assert (adm == k_out.view(torch.int16)[None]).any(0).all(), "K' not an admissible re-rotation"
    else:
        assert _same(k_out, _gather(k, idx)), "K' is not an exact gather"


def test_window_in_a_short_last_chunk():
    """The window straddles the last two chunks, and the short last chunk keeps fewer positions than it holds: its
    window positions compete for that chunk's budget, the lowest ones winning the tie."""
    S, w, L, r = 1031, 10, 256, 0.25  # last chunk [1024, 1031) keeps 5 of its 7 window positions
    k, v, q = inputs(1, 2, 2, S, 64, w, FP16, seed=13)
    k_out, v_out, idx, scores = native.finch_compress(k, v, q, w, r, L, True, None, True, True)
    want = chunked_topk(scores, w, L, r)
    assert torch.equal(idx.long(), want)
    assert (idx[..., -5:].long() == torch.arange(1024, 1029, device=DEV)).all()
    assert _same(k_out, _gather(k, idx)) and _same(v_out, _gather(v, idx))


def test_chunked_ties_and_short_last_chunk():
    """Planted ties (four distinct scores) through the caller-scores entry point, and a last chunk of one position."""
    S, w, L, r = 1031, 10, 256, 0.25
    k, v, _ = inputs(1, 3, 1, S, 64, w, FP16, seed=3)
    g = torch.Generator(device=DEV).manual_seed(5)
    scores = torch.randint(0, 4, (1, 3, S), generator=g, device=DEV).to(FP16)  # heavy ties
    k_out, v_out, idx = native.scores_compress_chunked(scores, k, v, r, L, None, True)
    want = chunked_topk(scores, 0, L, r)
    assert torch.equal(idx.long(), want)
    assert _same(k_out, _gather(k, idx)) and _same(v_out, _gather(v, idx))
    # a last chunk of one position
    S1 = 2 * 256 + 1
    k1, v1 = k[:, :, :S1], v[:, :, :S1]
    _, _, idx1 = native.scores_compress_chunked(scores[..., :S1], k1, v1, r, 256, None, True)
    assert torch.equal(idx1.long(), chunked_topk(scores[..., :S1], 0, 256, r))


def test_layouts_and_batch_independence():
    S, w, G = 2000, 50, 4
    k, v, q = inputs(2, 2, G, S, 128, w, BF16, seed=11)
    base = native.finch_compress(k, v, q, w, 0.5, 512, True, None, True, True)
    big = torch.randn(2, 4, S + 16, 136, device=DEV).to(BF16)
    big[:, 1:3, 8:8 + S, :128] = k
    ks = big[:, 1:3, 8:8 + S, :128]  # strided, sliced view
    out = native.finch_compress(ks, v, q, w, 0.5, 512, True, None, True, True)
    for a, b in zip(base, out):
        assert torch.equal(a, b)
    # a row's outputs do not depend on its batch; the window sentinel is the whole call's max + 1, so it may
    one = native.finch_compress(k[1:], v[1:], q[1:], w, 0.5, 512, True, None, True, True)
    for a, b in zip(base[:3], one[:3]):
        assert torch.equal(a[1:], b)
    assert torch.equal(base[3][1:, :, : S - w], one[3][..., : S - w])


def test_graph_capture():
    S, w = 4096, 100
    k, v, q = inputs(1, 8, 4, S, 128, w, BF16, seed=2)
    ref = native.finch_compress(k, v, q, w, 0.5, None, True, None, True, True)
    graphed = native.capture(lambda: native.finch_compress(k, v, q, w, 0.5, None, True, None, True, True))
    before = torch.cuda.memory_allocated()
    graphed.replay()
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == before
    for a, b in zip(ref, graphed.outputs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("D,G", [(96, 4), (256, 2), (64, 16)])
def test_fallback_shapes(D, G):
    S, w = 700, 33
    k, v, q = inputs(1, 2, G, S, D, w, BF16, seed=D)
    assert not finch_wide_head.finch_on_tensor_cores(D, G)
    got = finch_wide_head.finch_scores(k, q, w, True)
    assert_scores(got, k, q, w, True, f"fallback D{D} G{G}")


def test_press_and_pipeline_on_tiny_llama():
    model = tiny_gpu_llama()
    tok = word_tokenizer()
    press = FinchPress(0.5, chunk_length=None)
    press.update_model_and_tokenizer(model, tok)
    pipe = KVPressTextGenerationPipeline(model=model, tokenizer=tok, device=DEV)
    context = words(60, seed=1) + " <|finch_sep|> " + words(12, seed=3)
    out = pipe(context, question=words(5, seed=2), press=press, max_new_tokens=4)
    assert isinstance(out["answer"], str)
    assert press.window_size == 12


def test_permuted_and_strided_caches():
    """K and V as [B, S, H, D] caches permuted to [B, H, S, D], and as slices of wider rows: bitwise the contiguous
    call."""
    S, w = 1500, 37
    k, v, q = inputs(2, 4, 2, S, 128, w, BF16, seed=17)
    base = native.finch_compress(k, v, q, w, 0.5, 300, True, rope_inv_freq("theta10000", 128), True, True)
    kp = k.permute(0, 2, 1, 3).contiguous().permute(0, 2, 1, 3)
    vp = v.permute(0, 2, 1, 3).contiguous().permute(0, 2, 1, 3)
    wide = torch.zeros(2, 4, S, 256, device=DEV, dtype=BF16)
    wide[..., 64:192] = v
    for kk, vv in ((kp, vp), (k, wide[..., 64:192]), (kp, wide[..., 64:192])):
        out = native.finch_compress(kk, vv, q, w, 0.5, 300, True, rope_inv_freq("theta10000", 128), True, True)
        for a, b in zip(base, out):
            assert torch.equal(a, b)
    assert torch.equal(native.finch_score(kp, q, w), base[3])


def _raw_compress(k, v, q, w, L, ck, tk, n_kept, ws):
    p = native.make_problem(k, v, n_kept, q.shape[1])
    B, H, S, D = k.shape
    outs = (torch.empty(B, H, n_kept, D, device=DEV, dtype=k.dtype), torch.empty(B, H, n_kept, D, device=DEV,
            dtype=k.dtype), torch.empty(B, H, n_kept, device=DEV, dtype=torch.int32),
            torch.empty(B, H, S, device=DEV, dtype=k.dtype))
    native._enqueue("kvp_finch_compress", k.device, p, k, v, q, w, 1, L, ck, tk, None, *outs, ws, ws.numel())
    return outs


def test_exact_size_and_poisoned_workspaces():
    """A workspace of exactly kvp_workspace_bytes(KVP_SCORER_FINCH), filled with 0xFF, gives bitwise the usual result
    chunked and unchunked; 256 bytes less is refused for the largest window."""
    S, w = 3000, 100
    k, v, q = inputs(1, 2, 4, S, 128, w, BF16, seed=19)
    n_bytes = native.workspace_bytes(native.make_problem(k, v, S, q.shape[1]), native.SCORER_FINCH)
    ws = torch.full((n_bytes,), 0xFF, dtype=torch.uint8, device=DEV)
    for chunk in (None, 1024):
        L, ck, tk, n = native.chunk_counts(S, chunk, 0.5)
        want = native.finch_compress(k, v, q, w, 0.5, chunk, True, None, True, True)
        ws.fill_(0xFF)
        got = _raw_compress(k, v, q, w, L, ck, tk, n, ws)
        for a, b in zip(want, got):
            assert torch.equal(a, b)
    # the size covers the largest window, w = S - 1: such a call is refused one 256-byte region short
    _, _, q_big = inputs(1, 2, 4, S, 128, S - 1, BF16, seed=19)
    with pytest.raises(RuntimeError, match="workspace too small"):
        _raw_compress(k, v, q_big, S - 1, 0, 0, 0, S // 2, ws[: n_bytes - 256])


@pytest.mark.parametrize("D,G,L,rerotate", [(96, 4, None, True), (256, 2, 700, True), (64, 16, 700, False),
                                            (96, 4, None, False)])
def test_fallback_press_selection(D, G, L, rerotate):
    """The press on shapes the kernels do not instantiate: cuBLAS scores, then the sm_90a selection with the window
    forced (scores_compress / _rerotate / _chunked), checked against the selection of those scores."""
    from types import SimpleNamespace

    S, w = 2100, 30
    k, v, q = inputs(1, 2, G, S, D, w, BF16, seed=D + G)
    inv = rope_inv_freq("theta10000", D)
    press = FinchPress(0.5, chunk_length=L, rerotate_keys=rerotate)
    press.window_size = w
    press.window_queries = lambda *a: q
    module = SimpleNamespace(rotary_emb=SimpleNamespace(inv_freq=inv))
    k_out, v_out = press.compress(module, None, k, v, None, {})
    scores = finch_wide_head.finch_scores(k, q, w, True)
    idx = chunked_topk(scores, w, L or 0, 0.5)
    assert _same(v_out, _gather(v, idx))
    if rerotate:
        adm = rerotation_admissible(k, idx, inv).view(torch.int16)
        assert (adm == k_out.view(torch.int16)[None]).any(0).all()
    else:
        assert _same(k_out, _gather(k, idx))


# ---------------------------------------------------------------------------------------------------
# inputs and outputs past the 2 GiB and 4 GiB byte offsets
# ---------------------------------------------------------------------------------------------------
E31, E32 = (1 << 31) // 2, (1 << 32) // 2  # the boundaries in bf16 elements
FS, FD, FW, FG = 4096, 128, 200, 4
SD = FS * FD


def _far_inputs(arena):
    """K and V [1, 2, S, D] whose head 1 rows straddle byte 2^31 (head stride), q_window straddling byte 2^32, and
    contiguous copies of all three."""
    hs = E31 - SD // 2
    k = arena.as_strided((1, 2, FS, FD), (2 * hs, hs, FD, 1), 0)
    v = arena.as_strided((1, 2, FS, FD), (2 * hs, hs, FD, 1), SD)
    qn = 2 * FG * FW * FD
    q = arena[E32 - qn // 2: E32 + qn // 2].view(1, 2 * FG, FW, FD)
    g = torch.Generator(device=DEV).manual_seed(23)
    for t in (k, v, q):
        t.copy_(torch.randn(t.shape, generator=g, device=DEV))
    return k, v, q, E32 + qn // 2 + 4096


def _far(arena, at, shape, dtype=BF16):
    n = math.prod(shape) * torch.finfo(dtype).bits // 16
    return arena[at: at + n].view(dtype).view(shape), at + n + 4096


def _case_score(arena):
    k, v, q, at = _far_inputs(arena)
    scores, _ = _far(arena, at, (1, 2, FS))
    p = native.make_problem(k, k, 0, q.shape[1])
    native._enqueue("kvp_finch_score", k.device, p, k, q, FW, 1, scores, scorer=native.SCORER_FINCH)
    assert torch.equal(scores, native.finch_score(k.contiguous(), q.clone(), FW))


def _case_compress(arena):
    k, v, q, at = _far_inputs(arena)
    L, ck, tk, n = native.chunk_counts(FS, 1000, 0.5)
    at = E32 + (E32 // 4)  # outputs straddling byte 2^32 + 2^31 (6 GiB would not fit): past 4 GiB
    ko, at = _far(arena, at - n * FD, (1, 2, n, FD))
    vo, at = _far(arena, at, (1, 2, n, FD))
    inv = rope_inv_freq("theta10000", FD).to(DEV)
    p = native.make_problem(k, v, n, q.shape[1])
    native._enqueue("kvp_finch_compress", k.device, p, k, v, q, FW, 1, L, ck, tk, inv, ko, vo, None, None,
                    scorer=native.SCORER_FINCH)
    want = native.finch_compress(k.contiguous(), v.contiguous(), q.clone(), FW, 0.5, 1000, True, inv)
    assert torch.equal(ko, want[0]) and torch.equal(vo, want[1])


def _case_chunked(arena):
    k, v, q, at = _far_inputs(arena)
    scores = native.finch_score(k.contiguous(), q.clone(), FW)
    far_scores = arena[E31 + 2 * SD: E31 + 2 * SD + 2 * FS].view(1, 2, FS)  # past byte 2^31, clear of K and V
    far_scores.copy_(scores)
    L, ck, tk, n = native.chunk_counts(FS, 777, 0.5)
    ko, at = _far(arena, at, (1, 2, n, FD))
    vo, at = _far(arena, at, (1, 2, n, FD))
    p = native.make_problem(k, v, n)
    sstride = (ctypes.c_int64 * 2)(2 * FS, FS)
    native._enqueue("kvp_scores_compress_chunked", k.device, p, far_scores, sstride, L, ck, tk, k, v, None, ko, vo,
                    None, scorer=native.SCORER_FINCH)
    want = native.scores_compress_chunked(scores, k.contiguous(), v.contiguous(), 0.5, 777)
    assert torch.equal(ko, want[0]) and torch.equal(vo, want[1])


FAR_CASES = {"kvp_finch_score": _case_score, "kvp_finch_compress": _case_compress,
             "kvp_scores_compress_chunked": _case_chunked}


def test_every_finch_entry_point_has_a_far_case():
    import re
    from pathlib import Path

    header = (Path(__file__).resolve().parent.parent / "include" / "kvpress_b200.h").read_text()
    declared = set(re.findall(r"kvp_status\s+(kvp_(?:finch_\w+|scores_compress_chunked))\(", header))
    assert declared == set(FAR_CASES)


@pytest.mark.parametrize("name", sorted(FAR_CASES))
def test_far_offsets(name):
    need = (E32 + E32 // 4 + (1 << 26)) * 2
    if torch.cuda.mem_get_info()[0] < need + (2 << 30):
        pytest.skip("not enough free device memory for the 4.6 GiB arena")
    arena = torch.full((need // 2,), float("nan"), dtype=BF16, device=DEV)
    FAR_CASES[name](arena)
    torch.cuda.synchronize()
