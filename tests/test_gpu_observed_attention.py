"""ObservedAttention on the GPU: the sm_90a kernels (csrc/observed_attention.cu) against a float64 evaluation of their
definition (include/kvpress_b200.h, kvp_observed_attention_score), from the same 16-bit inputs, evaluated on the device
in blocks of query rows (no S x S tensor).

Bars, those of tests/test_gpu_scorer_sweep.py: every score within 1 ulp of the fp64 score rounded once (ex2.approx.ftz
may flush results below 2^-126); no row bias (|mean relative error| <= 8 u / sqrt(12 n) over rows of >= 500
normal-range positions). Compress keeps the lowest-index-ties top-n_kept of its own scores, which equal the score call's
bitwise, and returns exact gathers.
"""
import pytest
import torch
from transformers import DynamicCache

from oracle import press_oracle as O
from tests import observed_attention_backend as OB
from tests.gpu_support import (assert_compress, assert_vs_ref64, gpu_ids, _name, _native, oa_inputs, oa_ref64,
                               _sm_count, tiny_gpu_llama)

gpu = pytest.mark.gpu
DEV = "cuda:0"


def run(k, v, q, scaling, what, n_kept=None, bias=True):
    """score and compress of one problem, both checked against fp64; returns (scores, ref)."""
    nat = _native()
    S = k.shape[2]
    sc = nat.observed_attention_score(k, q, scaling)
    ref = oa_ref64(k, q, scaling)
    assert_vs_ref64(sc, ref, torch.zeros(S, dtype=torch.bool), what, ftz=True, bias=bias)
    assert torch.equal(nat.observed_attention_score(k, q, scaling), sc), f"{what}: two calls differ"
    n_kept = max(1, O.kept_count(S, 0.5)) if n_kept is None else n_kept
    k_out, v_out, idx, sc2 = nat.observed_attention_compress(k, v, q, scaling, n_kept, return_indices=True,
                                                             return_scores=True)
    assert torch.equal(sc2, sc), f"{what}: compress scores differ from the score path"
    assert_compress(k, v, k_out, v_out, idx, sc2, n_kept)
    return sc, ref


# --------------------------------------------------------------------------------------------------
# every instantiation, the edges of S and n_q, layouts
# --------------------------------------------------------------------------------------------------
SWEEP = [(dt, D, G) for dt in (torch.bfloat16, torch.float16) for D in (64, 128) for G in (1, 2, 3, 4, 5, 8)]


@gpu
@pytest.mark.parametrize("dtype,D,G", SWEEP, ids=[f"{_name(dt)}-d{D}-g{G}" for dt, D, G in SWEEP])
def test_instantiations(dtype, D, G):
    k, v, q = oa_inputs(1, 2, G, 1000, 1000, D, dtype, seed=G * 10 + D)
    run(k, v, q, D ** -0.5, f"obs {_name(dtype)} d{D} g{G}")


EDGES = [(S, n_q) for S in (1, 2, 127, 128, 129, 255, 256, 257, 1000, 4097, 16384)
         for n_q in sorted({S, max(1, S - 1), min(S, 130), min(S, 7), 1})]


@gpu
@pytest.mark.parametrize("S,n_q", EDGES, ids=[f"s{S}-nq{n}" for S, n in EDGES])
def test_sequence_and_query_edges(S, n_q):
    i = EDGES.index((S, n_q))
    dtype, D, G = SWEEP[(5 * i) % len(SWEEP)]  # spread the instantiations over the edges
    k, v, q = oa_inputs(1, 2, G, S, n_q, D, dtype, seed=i)
    run(k, v, q, D ** -0.5, f"obs {_name(dtype)} d{D} g{G} S{S} n_q{n_q}")


@gpu
def test_32k():
    k, v, q = oa_inputs(1, 2, 4, 32768, 32768, 128, torch.bfloat16, seed=32)
    run(k, v, q, 128 ** -0.5, "obs bf16 d128 g4 S32768")


@gpu
@pytest.mark.parametrize("layout", ["batch3", "strided", "transposed", "scaling"])
def test_layouts_and_scaling(layout):
    B, Hkv, G, S, D = (3 if layout == "batch3" else 2), 2, 4, 1500, 128
    k, v, q = oa_inputs(B, Hkv, G, S, S - 200, D, torch.bfloat16, seed=7)
    scaling = 0.3 if layout == "scaling" else D ** -0.5
    if layout == "strided":  # rows of D within rows of D + 64: consumed in place through the TMA map
        big = torch.zeros((B, Hkv, S, D + 64), dtype=k.dtype, device=DEV)
        big[..., :D] = k
        k = big[..., :D]
    elif layout == "transposed":  # a [B, S, Hkv, D] cache viewed as [B, Hkv, S, D]
        k = k.transpose(1, 2).contiguous().transpose(1, 2)
    sc, _ = run(k, v, q, scaling, f"obs {layout}")
    assert torch.equal(sc, _native().observed_attention_score(k.contiguous(), q, scaling))


@gpu
@pytest.mark.parametrize("regime", ["fewer", "equal", "more"])
def test_schedule_regimes(regime):
    """Items (R x 128-key tiles; with G = 1 also R x 128-query blocks) fewer than, equal to and more than the SMs."""
    sm = _sm_count()
    R = 4 if sm % 4 == 0 else 1
    tiles = {"fewer": sm // R - 1, "equal": sm // R, "more": 2 * sm // R + 1}[regime]
    S = tiles * 128
    items = R * -(-S // 128)
    assert (items < sm, items == sm, items > sm)[["fewer", "equal", "more"].index(regime)]
    k, v, q = oa_inputs(1, R, 1, S, S, 64, torch.float16, seed=tiles)
    run(k, v, q, 64 ** -0.5, f"obs schedule {regime} ({items} items, {sm} SMs)")


@gpu
def test_fp16_divisor_overflow():
    """S - s >= 65520 is inf in fp16: those first positions score exactly 0; the rest meet the 1-ulp bar."""
    S = 65600
    k, v, q = oa_inputs(1, 1, 1, S, S, 64, torch.float16, seed=3)
    sc = _native().observed_attention_score(k, q, 64 ** -0.5)
    zero = torch.arange(S, device=DEV) <= S - 65520
    assert int(zero.sum()) == 81
    assert (sc[..., zero] == 0).all() and not sc[..., zero].signbit().any()
    ref = oa_ref64(k, q, 64 ** -0.5)
    assert (ref[..., zero] == 0).all()
    assert_vs_ref64(sc, ref, torch.zeros(S, dtype=torch.bool), "obs fp16 S65600", ftz=True)


@gpu
def test_unsupported_shapes():
    nat = _native()
    k, _, q = oa_inputs(1, 2, 16, 300, 300, 128, torch.bfloat16, seed=1)
    with pytest.raises(RuntimeError, match="unsupported shape"):
        nat.observed_attention_score(k, q, 0.1)
    k, _, q = oa_inputs(1, 2, 2, 300, 300, 96, torch.bfloat16, seed=1)
    with pytest.raises(RuntimeError, match="unsupported shape"):
        nat.observed_attention_score(k, q, 0.1)


# --------------------------------------------------------------------------------------------------
# graph replay, memory (the torch GEMM fallback: tests/test_gpu_wide_head_sweep.py)
# --------------------------------------------------------------------------------------------------
@gpu
def test_replays_under_capture():
    nat = _native()
    k, v, q = oa_inputs(1, 4, 4, 3000, 3000, 128, torch.bfloat16, seed=9)
    eager = nat.observed_attention_compress(k, v, q, 128 ** -0.5, 1500, True, True)
    g = nat.capture(lambda: (nat.observed_attention_score(k, q, 128 ** -0.5),
                             *nat.observed_attention_compress(k, v, q, 128 ** -0.5, 1500, True, True)))
    q.copy_(torch.randn_like(q.float()).to(q.dtype))  # inputs updated in place
    out = g.replay()
    torch.cuda.synchronize()
    fresh = (nat.observed_attention_score(k, q, 128 ** -0.5),
             *nat.observed_attention_compress(k, v, q, 128 ** -0.5, 1500, True, True))
    assert all(torch.equal(a, b) for a, b in zip(out, fresh))
    assert not torch.equal(out[3], eager[2])


@gpu
def test_no_intermediate_at_32k():
    """Memory grows by no more than the workspace, the outputs and the query tensor: no S x S weights."""
    nat = _native()
    B, Hkv, G, S, D = 1, 8, 4, 32768, 128
    k, v, q = oa_inputs(B, Hkv, G, S, S, D, torch.bfloat16, seed=10)
    n_kept = S // 2
    p = nat.make_problem(k, v, n_kept, Hkv * G)
    ws = nat.workspace_bytes(p, nat.SCORER_OBSERVED_ATTENTION)
    nat._WS_CACHE.clear()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    out = nat.observed_attention_compress(k, v, q, D ** -0.5, n_kept, True, True)
    torch.cuda.synchronize()
    outputs = sum(t.numel() * t.element_size() for t in out if t is not None)
    grown = torch.cuda.max_memory_allocated() - before
    q_bytes = q.numel() * q.element_size()
    assert grown <= max(ws, 1 << 20) + outputs + q_bytes + (1 << 16), (grown, ws, outputs)
    assert grown < B * Hkv * G * S * S // 64  # a 64th of one layer's [B, Hq, S, S] bf16 weights


# --------------------------------------------------------------------------------------------------
# the press on a GPU tiny Llama (head_dim 64)
# --------------------------------------------------------------------------------------------------


def _checked_compress(monkeypatch, calls):
    """native.observed_attention_compress, checked on every call against the stand-in's scores on the same queries and
    keys (1 ulp) and against the canonical selection of its own scores."""
    nat = _native()
    real = nat.observed_attention_compress

    def checked(keys, values, q, scaling, n_kept, return_indices=False, return_scores=False):
        k_out, v_out, idx, sc = real(keys, values, q, scaling, n_kept, True, True)
        ref = OB.observed_attention_scores64(keys, q, scaling)
        assert_vs_ref64(sc, ref, torch.zeros(keys.shape[2], dtype=torch.bool), "press call", ftz=True, bias=False)
        assert_compress(keys, values, k_out, v_out, idx, sc, n_kept)
        calls.append(q.shape[2])
        return k_out, v_out, idx if return_indices else None, sc if return_scores else None

    monkeypatch.setattr(nat, "observed_attention_compress", checked)


@gpu
def test_press_and_decoding_press_on_a_tiny_llama(monkeypatch):
    from kvpress_b200 import DecodingPress, ObservedAttentionPress

    model, ids = tiny_gpu_llama(), gpu_ids()
    calls = []
    _checked_compress(monkeypatch, calls)
    cache = DynamicCache()
    with ObservedAttentionPress(compression_ratio=0.5)(model):
        model.model(input_ids=ids, past_key_values=cache)
    assert cache.get_seq_length() == 120 and calls == [240, 240]
    calls.clear()
    cache = DynamicCache()
    with DecodingPress(ObservedAttentionPress(), compression_interval=4, target_size=200)(model):
        model.model(input_ids=ids[:, :190], past_key_values=cache)
        for t in range(12):
            model.model(input_ids=ids[:, 190 + t:191 + t], past_key_values=cache)
    assert calls and set(calls) == {1} and cache.get_seq_length() <= 202


@gpu
def test_adakv_and_key_rerotation_run_under_sdpa():
    from kvpress_b200 import AdaKVPress, KeyRerotationPress, ObservedAttentionPress

    model, ids = tiny_gpu_llama(), gpu_ids()
    cache = DynamicCache()
    with AdaKVPress(ObservedAttentionPress(compression_ratio=0.5))(model):
        model.model(input_ids=ids, past_key_values=cache)
    attn = [layer.self_attn for layer in model.model.layers]
    assert cache.get_seq_length() == 240 and all(a.masked_key_indices is not None for a in attn)
    for a in attn:
        a.masked_key_indices = None
    cache = DynamicCache()
    with KeyRerotationPress(ObservedAttentionPress(compression_ratio=0.5))(model):
        out = model(input_ids=ids, past_key_values=cache).logits
    assert cache.get_seq_length() == 120 and torch.isfinite(out.float()).all()
