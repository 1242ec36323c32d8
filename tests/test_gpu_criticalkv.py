"""CriticalKV on the GPU: the sm_90a score kernel (csrc/criticalkv.cu) against a float64 evaluation of its definition
(include/kvpress_b200.h, kvp_criticalkv_score), from the same 16-bit inputs, evaluated on the device.

Bars, as in tests/test_gpu_scorer_sweep.py: every non-forced position within 1 ulp of the fp64 score rounded once; no
row bias (|mean relative error| <= 8 u / sqrt(12 n) over rows of >= 500 normal-range positions); the forced positions
are exactly the lowest-index-ties top-n_first of the base scores and hold finfo(dtype).max. Compress keeps the
top-n_kept of its own scores and returns exact gathers.
"""

import pytest
import torch
from transformers import DynamicCache

from oracle import press_oracle as O
from tests import criticalkv_backend
from tests.tiny_models import tiny_llama
from tests.gpu_support import ckv_assert_scores, ckv_inputs, _name, _native

gpu = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = [torch.bfloat16, torch.float16]
UNIT_ROUNDOFF = {torch.bfloat16: 2.0 ** -7, torch.float16: 2.0 ** -10}
BIAS_MIN_N = 500


def run_score(v, wo, base, eps, n_first, what, bias=True):
    native = _native()
    got = native.criticalkv_score(base, v, wo, eps, n_first)
    torch.cuda.synchronize()
    ckv_assert_scores(got, base, v, wo, eps, n_first, what, bias)
    return got


# --------------------------------------------------------------------------------------------------
# every instantiation: dtype x D, with every group-size regime
# --------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("G", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", DTYPES, ids=_name)
def test_instantiations(dtype, D, G):
    S = 1000
    v, wo, base = ckv_inputs(1, 2, G, S, D, 1000, dtype, seed=G * 10 + D)
    run_score(v, wo, base, 1e-4, 200, f"ckv {_name(dtype)} d{D} g{G}")


@gpu
@pytest.mark.parametrize("hidden", [4096, 1000, 64])
@pytest.mark.parametrize("dtype", DTYPES, ids=_name)
def test_hidden_sizes(dtype, hidden):
    """hidden a multiple of the 128-row Wo chunk, not one, and below one chunk: rows past hidden read as zero."""
    v, wo, base = ckv_inputs(1, 2, 4, 700, 128, hidden, dtype, seed=hidden)
    run_score(v, wo, base, 1e-4, 100, f"ckv {_name(dtype)} hidden {hidden}")


@gpu
@pytest.mark.parametrize("S", [1, 127, 128, 129, 255, 256, 257, 4097])
def test_sequence_lengths_and_batch(S):
    v, wo, base = ckv_inputs(3, 2, 2, S, 64, 512, torch.bfloat16, seed=S)
    run_score(v, wo, base, 1e-4, S // 3, f"ckv S {S} B 3")


@gpu
def test_llama8b_layer_rows_spread_over_every_sm():
    """The 8B layer shape at 8k: 256 items, so every CTA owns items of several rows."""
    v, wo, base = ckv_inputs(1, 8, 4, 8192, 128, 4096, torch.bfloat16, seed=8)
    run_score(v, wo, base, 1e-4, 2048, "ckv llama8b 8k")


@gpu
@pytest.mark.parametrize("layout", ["s_slice", "transposed", "wo_stride"])
def test_strided_operands_are_consumed_in_place(layout):
    native = _native()
    B, Hkv, G, S, D, hidden = 2, 4, 2, 600, 128, 700
    v, wo, base = ckv_inputs(B, Hkv, G, S, D, hidden, torch.bfloat16, seed=3)
    if layout == "s_slice":
        big = torch.randn((B, Hkv, S + 40, D), device=DEV).to(v.dtype)
        big[:, :, 17:17 + S] = v
        vv, ww = big[:, :, 17:17 + S], wo
    elif layout == "transposed":
        vv, ww = v.transpose(1, 2).contiguous().transpose(1, 2), wo  # [B, S, H, D] storage
    else:
        big = torch.randn((hidden, Hkv * G * D + 64), device=DEV).to(v.dtype)
        big[:, 32:32 + Hkv * G * D] = wo
        vv, ww = v, big[:, 32:32 + Hkv * G * D]
        assert ww.stride(0) > Hkv * G * D
    assert not vv.is_contiguous() or not ww.is_contiguous()
    got = native.criticalkv_score(base, vv, ww, 1e-4, 50)
    assert torch.equal(got, native.criticalkv_score(base, v, wo, 1e-4, 50))
    ckv_assert_scores(got, base, v, wo, 1e-4, 50, f"ckv {layout}")


@gpu
def test_base_scores_with_sentinels_and_strided_base():
    """Base scores of a wrapped press carry max + 1 on its forced positions; a broadcast-free strided base view."""
    v, wo, base = ckv_inputs(2, 2, 4, 900, 64, 512, torch.bfloat16, seed=4)
    base[..., :4] = (base.float().max() + 1).to(base.dtype)
    base[..., -64:] = (base.float().max() + 1).to(base.dtype)
    run_score(v, wo, base, 1e-4, 100, "ckv sentinels")
    wide = torch.zeros((2, 2, 1000), dtype=base.dtype, device=DEV)
    wide[..., :900] = base
    assert torch.equal(_native().criticalkv_score(wide[..., :900], v, wo, 1e-4, 100),
                       _native().criticalkv_score(base, v, wo, 1e-4, 100))


@gpu
def test_fp16_overflow_goes_to_inf():
    v, wo, base = ckv_inputs(1, 2, 2, 600, 128, 2048, torch.float16, seed=5, base_scale=60000.0)
    got = run_score(v, wo, base, 1e-4, 10, "ckv fp16 overflow", bias=False)
    assert torch.isinf(got).sum() > 100


@gpu
@pytest.mark.parametrize("n_first", [0, 1, 333, 600, 1000])
def test_forced_positions_are_the_top_n_first_of_base(n_first):
    v, wo, base = ckv_inputs(2, 2, 2, 1000, 64, 256, torch.float16, seed=6)
    base[0, 0, 100:300] = base[0, 0, 100]  # a long run of ties across the n_first threshold
    got = run_score(v, wo, base, 1e-4, n_first, f"ckv n_first {n_first}")
    assert int((got == torch.finfo(got.dtype).max).sum()) == 4 * n_first


@gpu
def test_two_calls_are_bitwise_equal():
    native = _native()
    v, wo, base = ckv_inputs(1, 8, 4, 20000, 128, 2048, torch.bfloat16, seed=7)
    a = native.criticalkv_score(base, v, wo, 1e-4, 5000)
    b = native.criticalkv_score(base, v, wo, 1e-4, 5000)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


@gpu
@pytest.mark.parametrize("n_first", [0, 150, 400])
@pytest.mark.parametrize("dtype", DTYPES, ids=_name)
def test_compress_keeps_the_top_of_its_own_scores(dtype, n_first):
    native = _native()
    B, Hkv, G, S, D, hidden = 2, 2, 4, 1000, 128, 1000
    v, wo, base = ckv_inputs(B, Hkv, G, S, D, hidden, dtype, seed=8)
    k = torch.randn_like(v)
    n_kept = 400
    k_out, v_out, idx, scores = native.criticalkv_compress(base, k, v, wo, 1e-4, n_first, n_kept, True, True)
    assert torch.equal(scores, native.criticalkv_score(base, v, wo, 1e-4, n_first))
    ckv_assert_scores(scores, base, v, wo, 1e-4, n_first, f"ckv compress {_name(dtype)} n_first {n_first}")
    want = O.select_lowest_index_ties(scores, n_kept)
    assert torch.equal(idx.long(), want)
    assert torch.equal(k_out, O.gather_rows(k, want)) and torch.equal(v_out, O.gather_rows(v, want))
    k2, v2, idx2, _ = native.criticalkv_compress(base, k, v, wo, 1e-4, n_first, n_kept, True)  # no scores output
    assert torch.equal(idx2, idx) and torch.equal(k2, k_out) and torch.equal(v2, v_out)


@gpu
def test_compress_replays_under_capture():
    native = _native()
    v, wo, base = ckv_inputs(1, 4, 2, 3000, 64, 1024, torch.bfloat16, seed=9)
    k = torch.randn_like(v)
    eager = native.criticalkv_compress(base, k, v, wo, 1e-4, 500, 1500, True, True)
    g = native.capture(lambda: native.criticalkv_compress(base, k, v, wo, 1e-4, 500, 1500, True, True))
    base.copy_(torch.rand_like(base.float()).to(base.dtype))  # inputs updated in place
    out = g.replay()
    torch.cuda.synchronize()
    fresh = native.criticalkv_compress(base, k, v, wo, 1e-4, 500, 1500, True, True)
    assert all(torch.equal(a, b) for a, b in zip(out, fresh))
    assert not torch.equal(out[2], eager[2])


@gpu
def test_no_intermediate_at_32k():
    """Memory grows by no more than the workspace and the outputs: nothing of size S x hidden is allocated."""
    native = _native()
    B, Hkv, G, S, D, hidden = 1, 8, 4, 32768, 128, 4096
    v, wo, base = ckv_inputs(B, Hkv, G, S, D, hidden, torch.bfloat16, seed=10)
    k = torch.randn_like(v)
    n_kept = S // 2
    p = native.make_problem(k, v, n_kept, Hkv * G)
    ws = native.workspace_bytes(p, native.SCORER_CRITICALKV)
    native._WS_CACHE.clear()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    out = native.criticalkv_compress(base, k, v, wo, 1e-4, n_kept // 2, n_kept, True, True)
    torch.cuda.synchronize()
    outputs = sum(t.numel() * t.element_size() for t in out if t is not None)
    grown = torch.cuda.max_memory_allocated() - before
    assert grown <= max(ws, 1 << 20) + outputs + (1 << 16), (grown, ws, outputs)
    assert grown < B * S * hidden * 2  # one head's [S, hidden] product alone would exceed this


# --------------------------------------------------------------------------------------------------
# the reference's evaluation registry on a GPU tiny Llama, against the same presses over the oracle stand-ins
# --------------------------------------------------------------------------------------------------
def _registry():
    from kvpress_b200 import CriticalAdaKVPress, CriticalKVPress, ExpectedAttentionPress, SnapKVPress

    return {
        "critical_snapkv": lambda r: CriticalKVPress(SnapKVPress(compression_ratio=r)),
        "critical_ea": lambda r: CriticalKVPress(ExpectedAttentionPress(compression_ratio=r, use_vnorm=False)),
        "critical_ada_snapkv": lambda r: CriticalAdaKVPress(SnapKVPress(compression_ratio=r)),
        "critical_ada_ea": lambda r: CriticalAdaKVPress(ExpectedAttentionPress(compression_ratio=r, use_vnorm=False)),
    }


def _run(model, press, ids):
    cache = DynamicCache()
    with press(model):
        model.model(input_ids=ids, past_key_values=cache)
    attns = [layer.self_attn for layer in model.model.layers]
    masks = [tuple(t.clone() for t in a.masked_key_indices) if getattr(a, "masked_key_indices", None) else None
             for a in attns]
    for a in attns:
        a.masked_key_indices = None
    return [(la.keys.clone(), la.values.clone()) for la in cache.layers], masks


@gpu
@pytest.mark.parametrize("name", ["critical_snapkv", "critical_ea", "critical_ada_snapkv", "critical_ada_ea"])
@pytest.mark.parametrize("head_dim", [64, 128])
def test_registry_presses_keep_the_same_rows_as_the_stand_ins(monkeypatch, name, head_dim):
    model = tiny_llama(dtype=torch.bfloat16, device=DEV, head_dim=head_dim, heads=8, kv_heads=2)
    model.config._attn_implementation = "sdpa"
    g = torch.Generator().manual_seed(11)
    ids = torch.stack([torch.randperm(250, generator=g)[:200] + 2 for _ in range(2)]).to(DEV)
    make = _registry()[name]
    ours, our_masks = _run(model, make(0.5), ids)
    with monkeypatch.context() as m:
        criticalkv_backend.install(m)
        theirs, their_masks = _run(model, make(0.5), ids)
    for (k1, v1), (k2, v2) in zip(ours, theirs):
        assert torch.equal(k1, k2) and torch.equal(v1, v2)
    for a, b in zip(our_masks, their_masks):
        assert (a is None) == (b is None)
        if a is not None:
            assert all(torch.equal(x, y) for x, y in zip(a, b))
    if "ada" in name:
        assert all(m is not None for m in our_masks) and ours[0][0].shape[2] == 200
    else:
        assert ours[0][0].shape[2] == 100
