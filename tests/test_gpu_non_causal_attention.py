"""NonCausalAttention on the GPU: the sm_90a kernels (csrc/non_causal_attention.cu) against a float64 evaluation of their
definition (include/kvpress_b200.h, kvp_non_causal_attention_score), from the same 16-bit inputs, evaluated on the device
in blocks of chunks (tests/non_causal_attention_backend.py).

Bars. z64 is the float64 score, u = 2^-24 the fp32 unit roundoff, ulp the spacing of the cache dtype at z64.
1. Every score is within 1 ulp of z64 rounded once, or |z - z64| <= ulp / 2 + E_s, where E_s bounds the kernel's fp32
   error at position s before the one rounding. So that the second arm cannot hide a fault, it may decide at most 1 % of
   a case's positions. (E_s itself is not small against the scores: with unscaled logits the worst-case dot-product
   error gamma tau below is about 1e-3 of a probability at head_dim 128, and the z-score multiplies a relative error of
   x by about (|z| + mean / std). E_s reaches 2^-5 to 2^-3 of a row's largest |z| on these inputs.)
2. No bias: over the positions with |z64| >= 1 of a row (at least 500 of them), the mean of (z - z64) / ulp is within
   8 / sqrt(12 n).
3. Compress keeps the lowest-index-ties top-n_kept of its own scores, which equal the score call's bitwise, and returns
   exact gathers.

E_s, derived from the code's operations. Let tau be the largest sum_d |q_d k_d| of any query row of the chunk (any head
of the group) and gamma = (D + 1) u: the products of 16-bit values are exact in fp32 and a wgmma accumulates D of them
in fp32, so every logit y carries |dy| <= gamma tau. Natural-log units below (log2(e) ln 2 = 1).
- P = ex2.approx(fma(y, log2 e, cb)), cb = -(m log2 e) - log2 Z. The row max m cancels between the exponent and Z up to
  its roundings, so the exponent carries the logit's own error, the normaliser's relative error
  dZ <= gamma tau + 4 u tau + 2^-22 + cs u (its exponents, ex2.approx's 2 ulp, its fp32 sum), and the roundings of
  m log2 e, log2f and the fma: dP <= gamma tau + dZ + 4 u tau + 4 u log2(cs) + 2^-22.
- A sums at most cs G such P in fp32 and divides by G: dA <= dP + (cs G + 2) u.
- ||v|| is an fp32 sum of D squares and a sqrt, (D + 2) u; x = A ||v|| adds u: eps_x = dA + (D + 4) u.
- pooled = ((x_{s-1} + x_s) + x_{s+1}) / 3 in fp32: dp_s <= sum of eps_x x over the three / 3 + 3 u pooled_s.
- mean and std from fp64 partials of those pooled values: |d mean| <= e mean(|pooled|), |d std| <= e rms(pooled), with
  e = max eps_x + 3 u. The z division runs in fp64.
E_s = 1.01 ((dp_s + |d mean|) / std + |z64| |d std| / std); the 1.01 covers the second-order terms.
"""
import math

import pytest
import torch
from transformers import DynamicCache

from oracle import press_oracle as O
from tests import non_causal_attention_backend as NB
from tests.gpu_support import (assert_compress, gpu_ids, _name, _native, nca_inputs, nca_ref, _sm_count,
                               tiny_gpu_llama, ulp16_diff, ulp_at)

gpu = pytest.mark.gpu
DEV = "cuda:0"
L2E = 1.0 / math.log(2.0)


def assert_vs_z64(got, z64, E, what: str, bias: bool = True) -> dict:
    """Bars 1 and 2 of the module docstring."""
    dtype = got.dtype
    z64 = z64.to(got.device)
    d = ulp16_diff(got, z64.to(dtype))
    near = (got.double() - z64).abs() <= ulp_at(z64, dtype) / 2 + E
    ok = (d <= 1) | near
    assert ok.all(), f"{what}: {int((~ok).sum())} positions beyond both bars (max {int(d.max())} ulp)"
    e_arm = int(((d > 1) & near).sum())
    assert e_arm <= max(1, d.numel() // 100), f"{what}: the E_s arm decides {e_arm} of {d.numel()} positions"
    stats = {"max_ulp": int(d.max()), "e_arm": e_arm}
    if bias:
        rel = (got.double() - z64) / ulp_at(z64, dtype)
        for r, m in zip(rel.reshape(-1, z64.shape[-1]), (z64.abs() >= 1).reshape(-1, z64.shape[-1])):
            n = int(m.sum())
            if n >= 500:
                assert abs(float(r[m].mean())) <= 8 / math.sqrt(12 * n), f"{what}: row bias {float(r[m].mean()):.3g}"
    return stats


def run(k, v, q, cs, what, n_kept=None, bias=True):
    """score and compress of one problem, both checked against fp64; returns (scores, z64)."""
    nat = _native()
    S = k.shape[2]
    sc = nat.non_causal_attention_score(k, v, q, cs)
    z64, E = nca_ref(k, v, q, cs)
    assert_vs_z64(sc, z64, E, what, bias=bias)
    assert torch.equal(nat.non_causal_attention_score(k, v, q, cs), sc), f"{what}: two calls differ"
    n_kept = max(1, O.kept_count(S, 0.5)) if n_kept is None else n_kept
    k_out, v_out, idx, sc2 = nat.non_causal_attention_compress(k, v, q, cs, n_kept, return_indices=True,
                                                               return_scores=True)
    assert torch.equal(sc2, sc), f"{what}: compress scores differ from the score path"
    assert_compress(k, v, k_out, v_out, idx, sc2, n_kept)
    return sc, z64


# --------------------------------------------------------------------------------------------------
# every instantiation, the edges of S, the padding quirk
# --------------------------------------------------------------------------------------------------
SWEEP = [(dt, D, cs, G) for dt in (torch.bfloat16, torch.float16) for D in (64, 128) for cs in (128, 256)
         for G in (1, 2, 3, 4, 5, 8)]


@gpu
@pytest.mark.parametrize("dtype,D,cs,G", SWEEP, ids=[f"{_name(dt)}-d{D}-cs{cs}-g{G}" for dt, D, cs, G in SWEEP])
def test_instantiations(dtype, D, cs, G):
    k, v, q = nca_inputs(1, 2, G, 1000, D, dtype, seed=G * 10 + D + cs)
    run(k, v, q, cs, f"nca {_name(dtype)} d{D} cs{cs} g{G}")


EDGES = sorted({(S, cs) for cs in (128, 256) for S in (1, 2, cs - 1, cs, cs + 1, 2 * cs - 1, 2 * cs + 1, 1000, 4097)})


@gpu
@pytest.mark.parametrize("S,cs", EDGES, ids=[f"s{S}-cs{cs}" for S, cs in EDGES])
def test_sequence_edges(S, cs):
    i = EDGES.index((S, cs))
    dtype, D, _, G = SWEEP[(7 * i) % len(SWEEP)]  # spread the instantiations over the edges
    k, v, q = nca_inputs(1, 2, G, S, D, dtype, seed=100 + i)
    run(k, v, q, cs, f"nca {_name(dtype)} d{D} g{G} S{S} cs{cs}", bias=S >= 1000)


@gpu
@pytest.mark.parametrize("S", [32768, 131072])
def test_long(S):
    """The Llama-3.1-8B layer shape (Hkv 8, G 4, D 128, cs 256) at 32k and 128k."""
    k, v, q = nca_inputs(1, 8, 4, S, 128, torch.bfloat16, seed=S % 1000)
    run(k, v, q, 256, f"nca llama8b S{S}", n_kept=O.kept_count(S, 0.7))


@gpu
@pytest.mark.parametrize("S", [1000, 4097, 511])
def test_padded_keys_take_the_mass(S):
    """Every logit of the last chunk's valid rows is below -100: the unmasked padded keys (logit 0) take their mass and
    the valid keys keep little beyond the padded query rows' pad / cs."""
    cs = 256
    k, v, q = nca_inputs(1, 2, 2, S, 128, torch.bfloat16, seed=S, negative_tail=True)
    sc, z64 = run(k, v, q, cs, f"nca negative tail S{S}", bias=False)
    x64 = NB.non_causal_attention_parts64(k, v, q, cs)
    s0 = (S - 1) // cs * cs
    pad = -(-S // cs) * cs - S
    vn = v[..., s0:, :].double().norm(dim=-1)
    assert torch.allclose(x64[..., s0:], pad / cs * vn, rtol=1e-6)


# --------------------------------------------------------------------------------------------------
# special cases of the global z-score
# --------------------------------------------------------------------------------------------------
@gpu
def test_constant_x_clamps_the_std():
    """Zero values: x and every pooled value are 0, the std is clamped to 1e-6 and every score is exactly 0."""
    nat = _native()
    B, Hkv, G, S, D = 1, 2, 2, 600, 64
    k = torch.full((B, Hkv, S, D), 0.5, device=DEV, dtype=torch.bfloat16)
    v = torch.zeros_like(k)
    q = torch.full((B, Hkv * G, S, D), 0.25, device=DEV, dtype=torch.bfloat16)
    sc = nat.non_causal_attention_score(k, v, q, 256)
    z64 = NB.non_causal_attention_scores64(k, v, q, 256)
    assert torch.equal(sc, z64.to(sc.dtype)) and (sc == 0).all()
    # one entry only: the unbiased std is 0 / 0, NaN as torch's
    k1, v1, q1 = k[:, :1, :1], v[:, :1, :1] + 1, q[:, :1, :1]
    one = nat.non_causal_attention_score(k1, v1, q1, 256)
    assert torch.isnan(one).all() and torch.isnan(NB.non_causal_attention_scores64(k1, v1, q1, 256)).all()


@gpu
def test_batch_couples_the_rows():
    """B = 3: mean and std run over the whole batch, so each sequence's scores depend on the others."""
    nat = _native()
    k, v, q = nca_inputs(3, 2, 4, 1500, 128, torch.bfloat16, seed=33)
    v[1] *= 4
    sc, _ = run(k, v, q, 256, "nca batch3")
    alone = nat.non_causal_attention_score(k[:1].contiguous(), v[:1].contiguous(), q[:1].contiguous(), 256)
    assert not torch.equal(alone[0], sc[0])


# --------------------------------------------------------------------------------------------------
# layouts: consumed in place, bitwise equal to contiguous copies
# --------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("layout", ["strided", "transposed", "slice"])
def test_layouts(layout):
    nat = _native()
    B, Hkv, G, S, D = 2, 2, 4, 1500, 128
    k, v, q = nca_inputs(B, Hkv, G, S, D, torch.bfloat16, seed=7)
    if layout == "strided":  # rows of D within rows of D + 64, for K and V
        kb = torch.zeros((B, Hkv, S, D + 64), dtype=k.dtype, device=DEV)
        vb = torch.zeros_like(kb)
        kb[..., :D], vb[..., :D] = k, v
        k, v = kb[..., :D], vb[..., :D]
    elif layout == "transposed":  # [B, S, Hkv, D] caches viewed as [B, Hkv, S, D]
        k = k.transpose(1, 2).contiguous().transpose(1, 2)
        v = v.transpose(1, 2).contiguous().transpose(1, 2)
    else:  # keys[..., 8:-4, :], as CompactorPress slices segments
        k, v, q = k[..., 8:-4, :], v[..., 8:-4, :], q[..., 8:-4, :]
        assert not k.is_contiguous() and nat._rows_ok(k)
    sc, _ = run(k, v, q, 256, f"nca {layout}")
    assert torch.equal(sc, nat.non_causal_attention_score(k.contiguous(), v.contiguous(), q.contiguous(), 256))


@gpu
@pytest.mark.parametrize("regime", ["fewer", "equal", "more"])
def test_schedule_regimes(regime):
    """Items (R x chunks) fewer than, equal to and more than the SMs."""
    sm = _sm_count()
    R = 4 if sm % 4 == 0 else 1
    chunks = {"fewer": sm // R - 1, "equal": sm // R, "more": 2 * sm // R + 1}[regime]
    S = chunks * 128 - 5
    items = R * -(-S // 128)
    assert (items < sm, items == sm, items > sm)[["fewer", "equal", "more"].index(regime)]
    k, v, q = nca_inputs(1, R, 2, S, 64, torch.float16, seed=chunks)
    run(k, v, q, 128, f"nca schedule {regime} ({items} items, {sm} SMs)")


@gpu
def test_unsupported_shapes_and_arguments():
    nat = _native()
    for G, D, cs in ((16, 128, 256), (2, 96, 256), (2, 128, 64), (2, 128, 512)):
        k, v, q = nca_inputs(1, 2, G, 300, D, torch.bfloat16, seed=1)
        with pytest.raises(RuntimeError, match="unsupported shape"):
            nat.non_causal_attention_score(k, v, q, cs)
    with pytest.raises(RuntimeError, match="bad argument"):
        nat.non_causal_attention_score(k, v, q, 0)


# --------------------------------------------------------------------------------------------------
# graph replay, workspace check, memory (the torch GEMM fallback: tests/test_gpu_wide_head_sweep.py)
# --------------------------------------------------------------------------------------------------
@gpu
def test_replays_under_capture_and_workspace_check():
    nat = _native()
    k, v, q = nca_inputs(1, 4, 4, 3000, 128, torch.bfloat16, seed=9)
    eager = nat.non_causal_attention_compress(k, v, q, 256, 1500, True, True)
    g = nat.capture(lambda: (nat.non_causal_attention_score(k, v, q, 256),
                             *nat.non_causal_attention_compress(k, v, q, 256, 1500, True, True)))
    q.copy_(torch.randn_like(q.float()).mul(1.3).to(q.dtype))  # inputs updated in place
    out = g.replay()
    torch.cuda.synchronize()
    fresh = (nat.non_causal_attention_score(k, v, q, 256), *nat.non_causal_attention_compress(k, v, q, 256, 1500,
                                                                                              True, True))
    assert all(torch.equal(a, b) for a, b in zip(out, fresh))
    assert not torch.equal(out[3], eager[2])
    p = nat.make_problem(k, v, 1500, q.shape[1])
    nat.workspace_check(p, nat.SCORER_NON_CAUSAL_ATTENTION, nat._workspace(p, nat.SCORER_NON_CAUSAL_ATTENTION,
                                                                          k.device))


@gpu
def test_no_intermediate_at_128k():
    """Memory grows by no more than the workspace and the outputs: no cs x cs tensor."""
    nat = _native()
    B, Hkv, G, S, D = 1, 8, 4, 131072, 128
    k, v, q = nca_inputs(B, Hkv, G, S, D, torch.bfloat16, seed=10)
    n_kept = S // 2
    p = nat.make_problem(k, v, n_kept, Hkv * G)
    ws = nat.workspace_bytes(p, nat.SCORER_NON_CAUSAL_ATTENTION)
    nat._WS_CACHE.clear()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    out = nat.non_causal_attention_compress(k, v, q, 256, n_kept, True, True)
    torch.cuda.synchronize()
    outputs = sum(t.numel() * t.element_size() for t in out if t is not None)
    grown = torch.cuda.max_memory_allocated() - before
    assert grown <= max(ws, 1 << 20) + outputs + (1 << 16), (grown, ws, outputs)


# --------------------------------------------------------------------------------------------------
# the press on GPU tiny Llamas (head_dim 64 and 128)
# --------------------------------------------------------------------------------------------------


@gpu
@pytest.mark.parametrize("head_dim", [64, 128])
def test_press_adakv_and_key_rerotation_on_a_tiny_llama(monkeypatch, head_dim):
    from kvpress_b200 import AdaKVPress, KeyRerotationPress, NonCausalAttnPress, native

    model, ids = tiny_gpu_llama(head_dim), gpu_ids()
    calls = []
    real = native.non_causal_attention_compress

    def checked(keys, values, q, cs, n_kept, return_indices=False, return_scores=False):
        k_out, v_out, idx, sc = real(keys, values, q, cs, n_kept, True, True)
        z64, E = nca_ref(keys, values, q, cs)
        assert_vs_z64(sc, z64, E, "press call", bias=False)
        assert_compress(keys, values, k_out, v_out, idx, sc, n_kept)
        calls.append(q.shape[2])
        return k_out, v_out, idx if return_indices else None, sc if return_scores else None

    monkeypatch.setattr(native, "non_causal_attention_compress", checked)
    cache = DynamicCache()
    with NonCausalAttnPress(compression_ratio=0.5, chunk_size=128)(model):
        model.model(input_ids=ids, past_key_values=cache)
    assert cache.get_seq_length() == 120 and calls == [240, 240]
    cache = DynamicCache()
    with AdaKVPress(NonCausalAttnPress(compression_ratio=0.5))(model):
        model.model(input_ids=ids, past_key_values=cache)
    attn = [layer.self_attn for layer in model.model.layers]
    assert cache.get_seq_length() == 240 and all(a.masked_key_indices is not None for a in attn)
    for a in attn:
        a.masked_key_indices = None
    cache = DynamicCache()
    with KeyRerotationPress(NonCausalAttnPress(compression_ratio=0.5))(model):
        out = model(input_ids=ids, past_key_values=cache).logits
    assert cache.get_seq_length() == 120 and torch.isfinite(out.float()).all()


@gpu
def test_decoding_press_fails_like_the_reference():
    from kvpress_b200 import DecodingPress, NonCausalAttnPress

    model, ids = tiny_gpu_llama(64), gpu_ids()
    cache = DynamicCache()
    with pytest.raises(AssertionError, match="only supports prefill"):
        with DecodingPress(NonCausalAttnPress(), compression_interval=4, target_size=100)(model):
            model.model(input_ids=ids[:, :190], past_key_values=cache)
            for t in range(8):
                model.model(input_ids=ids[:, 190 + t:191 + t], past_key_values=cache)
