"""kvp_cam_compress on an H100 against the float64 definition of tests/cam_backend.py, and CAMPress end to end.

Every case checks: the kept positions and the candidates exactly, K_out and the pruned running sum as exact gathers,
p_i against the float64 p_i to fp32 rounding of its window sum, and V_out within the header's bound of the float64 V
built with the kernel's own draws."""
import ctypes
import re
from pathlib import Path

import pytest
import torch

from kvpress_b200 import native
from tests import cam_backend as CB

pytestmark = pytest.mark.gpu
DEV = "cuda"
HEADER = Path(__file__).resolve().parent.parent / "include" / "kvpress_b200.h"
U = 2.0 ** -24


def _ulp(x: torch.Tensor, dtype) -> torch.Tensor:
    p, tiny = (8, 2.0 ** -133) if dtype == torch.bfloat16 else (11, 2.0 ** -24)
    _, e = torch.frexp(x)
    return torch.clamp(torch.pow(2.0, (e - p).double()), min=tiny)


def make(B, H, S, D, dtype, seed, scores_kind="randn"):
    g = torch.Generator(device=DEV).manual_seed(seed)
    keys = torch.randn(B, H, S, D, device=DEV, generator=g).to(dtype)
    values = torch.randn(B, H, S, D, device=DEV, generator=g).to(dtype)
    if scores_kind == "randn":
        scores = torch.randn(B, H, S, device=DEV, generator=g).to(dtype)
    elif scores_kind == "ties":
        scores = torch.randint(0, 2, (B, H, S), device=DEV, generator=g).to(dtype)
    else:  # NaN and inf rows among the scores
        scores = torch.randn(B, H, S, device=DEV, generator=g).to(dtype)
        scores[:, 0, ::7] = float("nan")
        scores[:, -1, 3::11] = float("inf")
        scores[:, -1, 5::13] = float("-inf")
    attn = torch.rand(B, H, S, device=DEV, generator=g) * 2
    return scores, keys, values, attn


def run(scores, keys, values, attn, n_kept, n_merge, budget, u, attn_out=None):
    B, H = keys.shape[:2]
    if attn_out is None:
        attn_out = torch.empty(B, H, n_kept, device=DEV)
    k, v, idx, midx, prob = native.cam_compress(scores, keys, values, attn, attn_out, n_merge, budget, u, n_kept,
                                                return_indices=True, return_plan=True)
    return k, v, attn_out, idx, midx, prob


def check(scores, keys, values, attn, n_kept, n_merge, budget, u, got):
    k, v, a_out, idx, midx, prob = got
    torch.cuda.synchronize()
    k64, v64, a64, kept, cand, p64 = CB.cam64(scores, keys, values, attn, n_merge, budget, u, n_kept, probs=prob)
    assert torch.equal(idx.long(), kept), "kept positions"
    assert torch.equal(midx.long(), cand), "candidates"
    assert torch.equal(k, k64) and torch.equal(a_out, a64.float()), "K / running sum gathers"
    tol = (min(budget, n_kept) + 4) * U * p64.abs() + 1e-37
    assert ((prob.double() - p64).abs() <= tol).all(), "merge probabilities"
    _, mag, *_ = CB.cam64(scores, keys, values.abs(), attn, n_merge, budget, u, n_kept, probs=prob)
    E = (n_merge + 2) * U * mag
    bound = _ulp(v64.abs() + E, keys.dtype) / 2 + E
    err = (v.double() - v64).abs()
    assert (err <= bound).all(), f"V_out off by {(err - bound).max().item()} beyond the bound"


def uniforms(B, H, n_merge, seed, kind="rand"):
    if kind == "zero":
        return torch.zeros(B, H, n_merge, device=DEV)
    if kind == "one":
        return torch.full((B, H, n_merge), 1 - 2.0 ** -24, device=DEV)
    return torch.rand(B, H, n_merge, device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("D", [64, 96, 128, 256])
@pytest.mark.parametrize("S", [2049, 2560])
def test_decoding_shapes(dtype, D, S):
    B, H, n_kept = 1, 8, 2048
    n_merge = min(512, S - n_kept)
    scores, keys, values, attn = make(B, H, S, D, dtype, S + D)
    u = uniforms(B, H, n_merge, D)
    check(scores, keys, values, attn, n_kept, n_merge, 32, u, run(scores, keys, values, attn, n_kept, n_merge, 32, u))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("S", [40000, 131584])
def test_long_caches(dtype, S):
    B, H, n_kept, n_merge = 1, 8, 2048, 512
    scores, keys, values, attn = make(B, H, S, 128, dtype, S)
    u = uniforms(B, H, n_merge, 1)
    check(scores, keys, values, attn, n_kept, n_merge, 32, u, run(scores, keys, values, attn, n_kept, n_merge, 32, u))


def test_streaming_scores_pile_every_candidate_on_the_first_recent_rows():
    """StreamingLLM: every evicted score is 0, so the candidates are the n_merge evicted positions before the recent
    window, they all share one t, and each of the first merge_budget recent rows receives all 512 of them."""
    B, H, S, n_kept, n_merge, sink = 1, 8, 131584, 2048, 512, 4
    _, keys, values, attn = make(B, H, S, 128, torch.bfloat16, 7)
    scores = torch.zeros(B, H, S, device=DEV, dtype=torch.bfloat16)
    scores[..., :sink] = 1
    scores[..., S - (n_kept - sink):] = 1
    u = uniforms(B, H, n_merge, 3, "zero")
    got = run(scores, keys, values, attn, n_kept, n_merge, 32, u)
    check(scores, keys, values, attn, n_kept, n_merge, 32, u, got)
    first_recent = S - (n_kept - sink)
    assert torch.equal(got[4][0].long().cpu(), torch.arange(first_recent - n_merge, first_recent))


@pytest.mark.parametrize("seed", range(12))
def test_small_caches(seed):
    g = torch.Generator().manual_seed(seed)
    S = int(torch.randint(3, 301, (1,), generator=g))
    n_kept = int(torch.randint(1, S, (1,), generator=g))
    n_merge = int(torch.randint(0, S - n_kept + 1, (1,), generator=g))
    budget = [1, 3, 32, S + 5][seed % 4]
    dtype = [torch.bfloat16, torch.float16][seed % 2]
    D = [8, 16, 64, 136][seed % 4]
    kind = ["randn", "ties", "nonfinite"][seed % 3]
    scores, keys, values, attn = make(2, 3, S, D, dtype, seed, kind)
    if seed % 5 == 0:
        attn[..., : S // 2] = 0  # zero running sums: 0 / 0 -> p = 0, and zero window means: x / 0 -> p = 1
    u = uniforms(2, 3, n_merge, seed, ["rand", "zero", "one"][seed % 3])
    check(scores, keys, values, attn, n_kept, n_merge, budget, u,
          run(scores, keys, values, attn, n_kept, n_merge, budget, u))


def test_batch_rows_equal_their_rows_alone_and_strided_views():
    B, H, S, D, n_kept, n_merge = 3, 4, 5000, 128, 2048, 512
    scores, keys, values, attn = make(B, H, S, D, torch.bfloat16, 11)
    u = uniforms(B, H, n_merge, 5)
    full = run(scores, keys, values, attn, n_kept, n_merge, 32, u)
    check(scores, keys, values, attn, n_kept, n_merge, 32, u, full)
    for b in range(B):
        alone = run(scores[b:b + 1], keys[b:b + 1], values[b:b + 1], attn[b:b + 1], n_kept, n_merge, 32, u[b:b + 1])
        for x, y in zip(full, alone):
            assert torch.equal(x[b:b + 1], y)
    # K / V as views of wider caches, the running sum and its output inside capacity buffers
    kk = torch.zeros(B, H, S + 8, 2 * D, device=DEV, dtype=keys.dtype)
    vv = torch.zeros(B, 2 * H, S, D, device=DEV, dtype=keys.dtype)
    kk[:, :, :S, :D] = keys
    vv[:, ::2] = values
    cap = torch.zeros(B, H, S + 300, device=DEV)
    cap[..., :S] = attn
    cap_out = torch.full((B, H, n_kept + 77), -1.0, device=DEV)
    strided = run(scores, kk[:, :, :S, :D], vv[:, ::2], cap[..., :S], n_kept, n_merge, 32, u, cap_out[..., :n_kept])
    for x, y in zip(full, strided):
        assert torch.equal(x, y)
    assert (cap_out[..., n_kept:] == -1).all()


def test_repeatable_graph_and_poisoned_workspace():
    B, H, S, D, n_kept, n_merge = 2, 8, 9000, 128, 2048, 512
    scores, keys, values, attn = make(B, H, S, D, torch.float16, 13)
    u = uniforms(B, H, n_merge, 2)
    a = [x.clone() for x in run(scores, keys, values, attn, n_kept, n_merge, 32, u)]
    b = run(scores, keys, values, attn, n_kept, n_merge, 32, u)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    out = torch.empty(B, H, n_kept, device=DEV)
    graph = native.capture(lambda: run(scores, keys, values, attn, n_kept, n_merge, 32, u, out))
    torch.cuda.synchronize()
    for _ in range(2):
        got = graph.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(x, y) for x, y in zip(a, got))
    # an exact-size workspace full of 0xFF
    p = native.make_problem(keys, values, n_kept)
    need = native.workspace_bytes(p, native.SCORER_CAM)
    ws = torch.full((need,), 0xFF, dtype=torch.uint8, device=DEV)
    k_out, v_out = torch.empty_like(a[0]), torch.empty_like(a[1])
    a_out = torch.empty(B, H, n_kept, device=DEV)
    idx = torch.empty(B, n_kept, dtype=torch.int32, device=DEV)
    st = (ctypes.c_int64 * 2)(S * H, S)
    ost = (ctypes.c_int64 * 2)(n_kept * H, n_kept)
    sst = (ctypes.c_int64 * 2)(S * H, S)
    rc = native.load().kvp_cam_compress(ctypes.byref(p), scores.data_ptr(), sst, keys.data_ptr(), values.data_ptr(),
                                        attn.data_ptr(), st, n_merge, 32, u.data_ptr(), k_out.data_ptr(),
                                        v_out.data_ptr(), a_out.data_ptr(), ost, idx.data_ptr(), None, None,
                                        ws.data_ptr(), need, native._stream())
    assert rc == 0
    torch.cuda.synchronize()
    assert torch.equal(k_out, a[0]) and torch.equal(v_out, a[1]) and torch.equal(a_out, a[2])
    assert torch.equal(idx, a[3])


# --------------------------------------------------------------------------------------------------
# inputs and outputs past the 4 GiB offset
# --------------------------------------------------------------------------------------------------
FAR = {"kvp_cam_compress"}


def test_every_cam_entry_point_has_a_far_offset_case():
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    assert set(re.findall(r"\b(kvp_cam_\w+)\s*\(", text)) == FAR


def test_far_offsets():
    """K, V, the running sum and every output placed past 4 GiB inside one buffer each."""
    B, H, S, D, n_kept, n_merge = 1, 8, 4096, 128, 2048, 512
    off = (4 << 30) + 4096  # bytes
    if torch.cuda.mem_get_info()[0] < 3 * off + (1 << 30):
        pytest.skip("not enough free device memory for three buffers past 4 GiB")
    scores, keys, values, attn = make(B, H, S, D, torch.bfloat16, 17)
    u = uniforms(B, H, n_merge, 9)
    want = run(scores, keys, values, attn, n_kept, n_merge, 32, u)
    torch.cuda.synchronize()
    big = torch.empty(off // 2 + keys.numel() * 2 + 64, dtype=torch.bfloat16, device=DEV)
    fk = big[off // 2: off // 2 + keys.numel()].view(keys.shape)
    fv = big[off // 2 + keys.numel(): off // 2 + 2 * keys.numel()].view(keys.shape)
    fk.copy_(keys)
    fv.copy_(values)
    del keys, values
    fa_buf = torch.empty(off // 4 + attn.numel() + n_kept * H + 64, dtype=torch.float32, device=DEV)
    fa = fa_buf[off // 4: off // 4 + attn.numel()].view(attn.shape)
    fa.copy_(attn)
    fo = fa_buf[off // 4 + attn.numel(): off // 4 + attn.numel() + n_kept * H].view(B, H, n_kept)
    got = run(scores, fk, fv, fa, n_kept, n_merge, 32, u, fo)
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(want, got))


# --------------------------------------------------------------------------------------------------
# the per-step running sum and the press
# --------------------------------------------------------------------------------------------------
def test_running_sum_over_300_steps():
    from kvpress_b200.presses.cam_press import RunningAttention

    B, H, Hq, D, S0 = 1, 4, 16, 128, 700
    g = torch.Generator(device=DEV).manual_seed(3)
    keys = torch.randn(B, H, S0 + 300, D, device=DEV, generator=g).to(torch.bfloat16)
    state = RunningAttention(B, H, S0, DEV)
    ref = torch.zeros(B, H, S0 + 300, dtype=torch.float64, device=DEV)
    slack = torch.zeros_like(ref)
    ptrs = {state.buf.data_ptr()}
    for step in range(300):
        S = S0 + step + 1
        q = torch.randn(B, Hq, D, device=DEV, generator=g).to(torch.bfloat16)
        k = keys[:, :, :S]
        state.add(native.expected_attention_score(k, k, q, None, 0.0, 0, False))
        logits = torch.einsum("bhd,bhsd->bhs", q.double(), k.double().repeat_interleave(Hq // H, 1)) / D ** 0.5
        p = logits.softmax(-1).view(B, H, Hq // H, S).mean(2)
        ref[..., :S] += p
        slack[..., :S] += p * 2.0 ** -7 + 1e-7 * p.amax(-1, keepdim=True)
        ptrs.add(state.buf.data_ptr())
    assert state.length == S0 + 300 and state.buf.shape[2] == 2 * S0
    assert len(ptrs) == 2  # the first step grows past the initial capacity, every later step reuses the buffer
    assert ((state.view().double() - ref).abs() <= slack).all()


@pytest.mark.parametrize("name", ["knorm", "streaming", "tova", "prefill_decoding"])
def test_presses_on_a_tiny_bf16_llama(name):
    from kvpress_b200 import (CAMPress, KnormPress, KVPressTextGenerationPipeline, PrefillDecodingPress,
                              StreamingLLMPress, TOVAPress)
    from tests.tiny_models import tiny_model, word_tokenizer, words

    model = tiny_model(dtype=torch.bfloat16, device=DEV, head_dim=64)
    pipe = KVPressTextGenerationPipeline(model=model, tokenizer=word_tokenizer(), device=DEV)
    target, interval = 48, 3
    make = {"knorm": lambda: CAMPress(KnormPress(), interval, target),
            "streaming": lambda: CAMPress(StreamingLLMPress(), interval, target),
            "tova": lambda: CAMPress(TOVAPress(), interval, target),
            "prefill_decoding": lambda: PrefillDecodingPress(KnormPress(0.6), CAMPress(KnormPress(), interval, target))}
    from transformers import DynamicCache

    cache = DynamicCache()
    torch.manual_seed(0)
    pipe(words(120, seed=1), question=words(6, seed=2), press=make[name](), cache=cache, max_new_tokens=15)
    for la in cache.layers:
        assert target <= la.keys.shape[2] <= target + interval - 1
