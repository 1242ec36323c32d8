"""MergingPress on the GPU: the sm_90a kernels (csrc/merging.cu) against a float64 evaluation of their definition
(include/kvpress_b200.h, kvp_merging_compress) from the same 16-bit inputs, on the device (tests/merging_backend.py).

With u = 2^-24 the fp32 unit roundoff, the kernel's similarity of evicted slot e and kept slot t is within
    E(e, t) = 1.01 ((D + 2) u sum_d |k_ed k_td| / (n_e n_t) + 24 u |sim64(e, t)|)
of the float64 similarity: exact products, fp32 accumulation of D terms, and two norms (an fp32 sum of squares over
8-element FMA chains and a 32-lane butterfly, a square root and a reciprocal) plus two scalings, each at most 10 u.
- target: the kernel's target is the float64 argmax, or its float64 similarity lies within E(e, target) + E(e, argmax)
  of the maximum. A NaN maximum is matched exactly (the first NaN column). sim_out is within E(e, target) of
  sim64(e, target).
- the gate: the set of merged evicted rows is the one torch.quantile gives on the kernel's own sim_out, so the
  kernel's threshold decides every entry exactly as torch's does.
- V_out: with the kernel's own targets and similarities, the float64 merge v64 rounded once is within 1 ulp of V_out,
  or within ulp(|v64| + E_v) + E_v where the fp32 sums cancel, on at most 1 % of the positions. With n contributions,
  the weights' fp32 relative error (two norms, the quotient) at most 32 u and A = |V[t]| + sum w |V[e]|:
  E_v = 1.01 u ((n + 1) A + 32 sum w |V[e]| + |v64| ((n + 1)(1 + sum w) + 32 sum w)) / (1 + sum w) + u |v64|.
  Kept rows that take no contribution are V[kept] bit for bit.
"""
import pytest
import torch
from transformers import DynamicCache

from oracle import press_oracle as O
from tests import cpu_backend, merging_backend as MB
from tests.gpu_support import _native, gpu_ids, tiny_gpu_llama, ulp_at

gpu = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24
DTYPES = [torch.bfloat16, torch.float16]


def inputs(B, H, S, D, dtype, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    k = (torch.randn(B, H, S, D, generator=g, device=DEV) * scale).to(dtype)
    v = torch.randn(B, H, S, D, generator=g, device=DEV).to(dtype)
    return k, v


def random_kept(B, H, S, n_kept, seed):
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    return torch.rand(B, H, S, generator=g, device=DEV).argsort(dim=-1)[..., :n_kept].sort(dim=-1).values.int()


def sim_bound(keys, kept, ev_rows=None):
    """(sim64, E) [B, H, n_evict (or the rows `ev_rows` of it), n_kept]."""
    ev = MB.complement(kept, keys.shape[2])
    if ev_rows is not None:
        ev = ev[..., ev_rows]
    k = keys.double()
    kk = k.gather(2, kept.long().unsqueeze(-1).expand(-1, -1, -1, k.shape[-1]))
    ke = k.gather(2, ev.unsqueeze(-1).expand(-1, -1, -1, k.shape[-1]))
    nk, ne = kk.norm(dim=-1).clamp(min=MB.EPS), ke.norm(dim=-1).clamp(min=MB.EPS)
    den = ne.unsqueeze(-1) * nk.unsqueeze(-2)
    sim = (ke @ kk.transpose(-1, -2)) / den
    E = 1.01 * ((k.shape[-1] + 2) * U * (ke.abs() @ kk.abs().transpose(-1, -2)) / den + 24 * U * sim.abs())
    return sim, E


def assert_plan(keys, kept, target, sim_out, ev_rows=None):
    """The kernel's targets and similarities against the float64 ones (module docstring)."""
    sim64, E = sim_bound(keys, kept, ev_rows)
    if ev_rows is not None:
        target, sim_out = target[..., ev_rows], sim_out[..., ev_rows]
    t = target.long()
    max64, arg64 = sim64.max(dim=-1)
    nan = max64.isnan()
    assert torch.equal(t[nan], arg64[nan]), "a NaN maximum goes to the first NaN column"
    assert not sim_out[~nan].isnan().any()
    at = sim64.gather(-1, t.unsqueeze(-1)).squeeze(-1)
    e_t = E.gather(-1, t.unsqueeze(-1)).squeeze(-1)
    e_a = E.gather(-1, arg64.unsqueeze(-1)).squeeze(-1)
    ok = nan | (t == arg64) | (at >= max64 - e_t - e_a)
    assert ok.all(), f"{int((~ok).sum())} targets are not the float64 argmax within the bound"
    assert ((sim_out.double() - at).abs()[~nan] <= e_t[~nan] + U * at.abs()[~nan]).all()
    return float((t != arg64)[~nan].float().mean()) if (~nan).any() else 0.0


def value_bound(values, kept, target, sim_out, ok, v64):
    """E_v of the module docstring, [B, H, n_kept, D]."""
    D = values.shape[-1]
    ev = MB.complement(kept, values.shape[2])
    vk = values.double().gather(2, kept.long().unsqueeze(-1).expand(-1, -1, -1, D))
    ve = values.double().gather(2, ev.unsqueeze(-1).expand(-1, -1, -1, D))
    tn, en = vk.norm(dim=-1), ve.norm(dim=-1)
    w = sim_out.double().clamp(min=0) * ok.double() * en / (en + tn.gather(2, target.long()) + MB.EPS)
    t4 = target.long().unsqueeze(-1).expand(-1, -1, -1, D)
    wv = torch.zeros_like(vk).scatter_add_(2, t4, w.unsqueeze(-1) * ve.abs())
    sw = torch.zeros_like(tn).scatter_add_(2, target.long(), w).unsqueeze(-1)
    n = torch.zeros_like(tn).scatter_add_(2, target.long(), torch.ones_like(w)).unsqueeze(-1)
    a = vk.abs() + wv
    q = v64.abs()
    return 1.01 * U * (((n + 1) * a + 32 * wv + q * ((n + 1) * (1 + sw) + 32 * sw)) / (1 + sw) + q)


def assert_values(values, kept, target, sim_out, thr, frac, v_out):
    """V_out against the float64 merge on the kernel's own plan, the gate by torch.quantile on sim_out."""
    ok = MB.gate(sim_out, thr, frac)
    v64 = MB.merged_values64(values, kept, target, sim_out.double(), ok)
    vk = values.gather(2, kept.long().unsqueeze(-1).expand(-1, -1, -1, values.shape[-1]))
    acc_w = torch.zeros(kept.shape, dtype=torch.float64, device=DEV)
    w = sim_out.double().clamp(min=0) * ok.double()
    acc_w.scatter_add_(2, target.long(), torch.where(w.isnan(), torch.ones_like(w), w))
    untouched = ~(acc_w > 0)
    assert torch.equal(v_out[untouched].view(torch.int16), vk[untouched].view(torch.int16)), "unmerged rows are copied"
    nanrow = v64.isnan()
    assert torch.equal(nanrow, v_out.isnan())
    assert_close16(v_out, v64, value_bound(values, kept, target, sim_out, ok, v64))
    return int((~untouched).sum())


def assert_close16(got, v64, E):
    """Within 1 ulp of v64, or within ulp(|v64| + E) + E on at most 1 % of the positions (NaN where v64 is NaN)."""
    fin = ~v64.isnan()
    diff = (got.double() - v64).abs()[fin]
    one = diff <= ulp_at(v64[fin], got.dtype)
    bound = diff <= ulp_at(v64[fin].abs() + E[fin], got.dtype) + E[fin]
    assert (one | bound).all(), float((diff / ulp_at(v64[fin], got.dtype)).max())
    assert (~one).float().mean() <= 0.01, float((~one).float().mean())


def check_merge(k, v, kept, thr=0.0, frac=1.0, ev_rows=None):
    nat = _native()
    v_out, target, sim = nat.merging_merge(k, v, kept, thr, frac, return_plan=True)
    torch.cuda.synchronize()
    assert target.shape == sim.shape == (*k.shape[:2], k.shape[2] - kept.shape[2])
    assert ((target >= 0) & (target < kept.shape[2])).all()
    moved = assert_plan(k, kept, target, sim, ev_rows)
    merged = assert_values(v, kept, target, sim, thr, frac, v_out) if ev_rows is None else None
    return v_out, target, sim, moved, merged


# --------------------------------------------------------------------------------------------------
# every instantiation: dtype x panel count
# --------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("D", [8, 64, 72, 96, 128, 192, 256])
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_instantiations(dtype, D):
    k, v = inputs(2, 3, 700, D, dtype, seed=D)
    kept = random_kept(2, 3, 700, 300, seed=D)
    _, _, _, moved, merged = check_merge(k, v, kept)
    assert moved <= 0.01 and merged > 100


@gpu
@pytest.mark.parametrize("n_kept,n_evict", [(1, 1), (1, 200), (63, 65), (64, 64), (65, 63), (127, 129), (128, 128),
                                            (129, 127), (255, 257), (300, 1), (1, 300), (700, 0), (256, 1000)])
def test_tile_edges(n_kept, n_evict):
    S = n_kept + n_evict
    k, v = inputs(1, 2, S, 128, torch.bfloat16, seed=S)
    kept = random_kept(1, 2, S, n_kept, seed=n_kept)
    if n_evict == 0:
        v_out, target, sim = _native().merging_merge(k, v, kept, 0.0, 1.0, return_plan=True)
        assert target.numel() == 0 and torch.equal(v_out, v)
        return
    check_merge(k, v, kept)


@gpu
@pytest.mark.parametrize("frac", [1.0, 0.75, 0.3, 0.05])
@pytest.mark.parametrize("thr", [0.0, 0.1, 0.35, 1.0])
def test_gate(thr, frac):
    """Thresholds up to 1 and fractions down to 0.05, on keys with a shared component so that many similarities pass;
    the quantile's order statistics are exact integers of rank at some fractions and interpolated at others."""
    k, v = inputs(2, 2, 900, 64, torch.float16, seed=7)
    k = (k.float() + 1.5 * torch.randn(2, 2, 1, 64, device=DEV)).to(torch.float16)
    kept = random_kept(2, 2, 900, 401, seed=3)
    check_merge(k, v, kept, thr, frac)


@gpu
def test_quantile_of_minus_inf_statistics_merges_nothing():
    """q = 0.25 over rows where most similarities fail the threshold: both order statistics are -inf, the threshold is
    NaN and the row merges nothing, as torch.quantile makes it."""
    k, v = inputs(1, 2, 400, 64, torch.bfloat16, seed=9)
    kept = random_kept(1, 2, 400, 200, seed=9)
    v_out, target, sim, _, merged = check_merge(k, v, kept, 0.6, 0.75)
    vk = v.gather(2, kept.long().unsqueeze(-1).expand(-1, -1, -1, 64))
    assert (sim < 0.6).float().mean() > 0.75 and merged == 0 and torch.equal(v_out, vk)


# --------------------------------------------------------------------------------------------------
# degenerate inputs, ties
# --------------------------------------------------------------------------------------------------
@gpu
def test_planted_ties_go_to_the_lowest_slot():
    """Kept slots 5, 9 and 40 of every row hold the same key; evicted rows that are positive multiples of it have three
    exactly tied maxima and must target slot 5."""
    k, v = inputs(2, 2, 500, 128, torch.bfloat16, seed=11)
    kept = random_kept(2, 2, 500, 200, seed=11)
    ev = MB.complement(kept, 500)
    base = torch.randn(2, 2, 1, 128, device=DEV)
    for b in range(2):
        for h in range(2):
            for t in (5, 9, 40):
                k[b, h, kept[b, h, t]] = base[b, h, 0].to(k.dtype)
            for i, scale in enumerate((1.0, 2.0, 0.5, 4.0)):
                k[b, h, ev[b, h, 10 * i]] = (base[b, h, 0] * scale).to(k.dtype)
    _, target, _, _, _ = check_merge(k, v, kept)
    assert (target[..., [0, 10, 20, 30]] == 5).all()


@gpu
def test_zero_nan_and_inf_rows():
    """Zero keys target slot 0 with similarity 0; a NaN kept key is the target of every evicted row and leaves its own
    value unmerged; an inf evicted key targets slot 0 with a NaN similarity; a NaN evicted value leaves its target as it
    was."""
    k, v = inputs(1, 4, 300, 64, torch.bfloat16, seed=13)
    kept = random_kept(1, 4, 300, 120, seed=13)
    ev = MB.complement(kept, 300)
    k[0, 0, ev[0, 0, :20]] = 0                      # zero evicted keys
    k[0, 0, kept[0, 0, 0]] = 0                      # a zero kept key
    k[0, 1, kept[0, 1, 7], 3] = float("nan")        # a NaN kept key
    k[0, 2, ev[0, 2, 4], 0] = float("inf")          # an inf evicted key
    v[0, 3, ev[0, 3, 2], 1] = float("nan")          # a NaN evicted value, whose key is kept slot 5's
    k[0, 3, ev[0, 3, 2]] = k[0, 3, kept[0, 3, 5]]
    v_out, target, sim, _, _ = check_merge(k, v, kept)
    assert (target[0, 0, :20] == 0).all() and (sim[0, 0, :20] == 0).all()
    assert (target[0, 1] == 7).all() and sim[0, 1].isnan().all()
    assert torch.equal(v_out[0, 1, 7].view(torch.int16), v[0, 1, kept[0, 1, 7]].view(torch.int16))
    assert target[0, 2, 4] == 0 and sim[0, 2, 4].isnan()
    # its norm, and so its weight, is NaN: its target's weight sum is NaN and that row is left as it was
    assert target[0, 3, 2] == 5 and not v_out[0, 3].isnan().any()
    assert torch.equal(v_out[0, 3, 5].view(torch.int16), v[0, 3, kept[0, 3, 5]].view(torch.int16))


# --------------------------------------------------------------------------------------------------
# layouts, many rows, schedules, long rows and memory
# --------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("layout", ["slice_along_s", "transposed_bshd", "every_other_head"])
def test_layouts(layout):
    k, v = inputs(2, 4, 640, 128, torch.bfloat16, seed=17)
    if layout == "slice_along_s":
        k, v = k[:, :, 20:-20], v[:, :, 20:-20]
    elif layout == "transposed_bshd":
        k, v = k.transpose(1, 2).contiguous().transpose(1, 2), v.transpose(1, 2).contiguous().transpose(1, 2)
    else:
        k, v = k[:, ::2], v[:, ::2]
    kept = random_kept(*k.shape[:3], 250, seed=17)
    v_out = check_merge(k, v, kept)[0]
    assert torch.equal(v_out, _native().merging_merge(k.contiguous(), v.contiguous(), kept, 0.0, 1.0)[0])


@gpu
def test_thousands_of_rows_and_the_batch():
    """3000 rows (more items than the persistent grid holds in any regime), and a batch equals its rows run alone."""
    k, v = inputs(375, 8, 200, 64, torch.bfloat16, seed=19)
    kept = random_kept(375, 8, 200, 90, seed=19)
    v_out, target, sim, _, _ = check_merge(k, v, kept, 0.1, 0.75)
    nat = _native()
    for b in (0, 200, 374):
        vo, t, s = nat.merging_merge(k[b:b + 1], v[b:b + 1], kept[b:b + 1], 0.1, 0.75, return_plan=True)
        assert torch.equal(vo, v_out[b:b + 1]) and torch.equal(t, target[b:b + 1]) and torch.equal(s, sim[b:b + 1])


@gpu
@pytest.mark.parametrize("S", [4096, 20000])
def test_schedule_regimes_and_determinism(S):
    """Fewer items than SMs, then many per SM; two calls are bitwise equal."""
    k, v = inputs(1, 2 if S == 4096 else 8, S, 128, torch.bfloat16, seed=S)
    kept = random_kept(*k.shape[:3], S // 2, seed=S)
    rows = torch.arange(0, S - S // 2, 97, device=DEV)
    a = check_merge(k, v, kept, 0.0, 0.75, ev_rows=rows)
    b = _native().merging_merge(k, v, kept, 0.0, 0.75, return_plan=True)
    for x, y in zip(a[:3], b):
        assert torch.equal(x.view(torch.int16) if x.dtype == torch.bfloat16 else x,
                           y.view(torch.int16) if y.dtype == torch.bfloat16 else y)
    assert_values(v, kept, b[1], b[2], 0.0, 0.75, b[0])


@gpu
def test_128k_row_within_the_workspace():
    """A Llama-3.1-8B layer at 128k, ratio 0.5: the reference's similarity tensor would take 137 GB. Here the device
    memory grows by the workspace and the outputs only; a sample of evicted rows is checked against float64."""
    nat = _native()
    S, n_kept = 131072, 65536
    k, v = inputs(1, 8, S, 128, torch.bfloat16, seed=23)
    kept = random_kept(1, 8, S, n_kept, seed=23)
    p = nat.make_problem(k, v, n_kept)
    ws = nat.workspace_bytes(p, nat.SCORER_MERGING)
    torch.cuda.synchronize()
    nat._WS_CACHE.clear()
    torch.cuda.empty_cache()
    before = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    v_out, target, sim = nat.merging_merge(k, v, kept, 0.0, 1.0, return_plan=True)
    torch.cuda.synchronize()
    outputs = v_out.numel() * 2 + target.numel() * 8
    assert torch.cuda.max_memory_allocated() - before <= max(ws, 1 << 20) + outputs + (4 << 20)
    rows = torch.randperm(S - n_kept, device=DEV)[:48]
    for h in range(8):
        assert_plan(k[:, h:h + 1], kept[:, h:h + 1], target[:, h:h + 1], sim[:, h:h + 1], ev_rows=rows)


# --------------------------------------------------------------------------------------------------
# the compress call, graphs
# --------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_compress_is_selection_then_merge(dtype):
    nat = _native()
    k, v = inputs(2, 4, 1500, 128, dtype, seed=29)
    scores = torch.randn(2, 4, 1500, device=DEV).to(dtype)
    k_out, v_out, idx, target, sim = nat.merging_compress(scores, k, v, 0.0, 1.0, 700, return_indices=True,
                                                          return_plan=True)
    torch.cuda.synchronize()
    want_idx = O.select_lowest_index_ties(scores.cpu(), 700).to(DEV)
    assert torch.equal(idx.long(), want_idx) and torch.equal(k_out, O.gather_rows(k, want_idx.long()))
    v2, t2, s2 = nat.merging_merge(k, v, idx, 0.0, 1.0, return_plan=True)
    assert torch.equal(v_out, v2) and torch.equal(target, t2) and torch.equal(sim, s2)
    assert_plan(k, idx, target, sim)
    assert_values(v, idx, target, sim, 0.0, 1.0, v_out)
    # without the optional outputs
    k3, v3, i3, t3, s3 = nat.merging_compress(scores, k, v, 0.0, 1.0, 700)
    assert i3 is None and t3 is None and torch.equal(v3, v_out) and torch.equal(k3, k_out)


@gpu
def test_graph_capture_replays_the_call():
    nat = _native()
    k, v = inputs(1, 8, 3000, 128, torch.bfloat16, seed=31)
    scores = torch.randn(1, 8, 3000, device=DEV).to(torch.bfloat16)
    eager = nat.merging_compress(scores, k, v, 0.1, 0.75, 1500)
    g = nat.capture(lambda: nat.merging_compress(scores, k, v, 0.1, 0.75, 1500))
    out = g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[0], eager[0]) and torch.equal(out[1], eager[1])
    k.copy_(inputs(1, 8, 3000, 128, torch.bfloat16, seed=32)[0])
    out = g.replay()
    want = nat.merging_compress(scores, k, v, 0.1, 0.75, 1500)
    torch.cuda.synchronize()
    assert torch.equal(out[1], want[1])


# --------------------------------------------------------------------------------------------------
# the press, alone and under wrappers, on a tiny Llama: every merge it asks for is checked as above
# --------------------------------------------------------------------------------------------------
@pytest.fixture
def calls(monkeypatch):
    nat = _native()
    real, seen = nat.merging_compress, []

    def recording(scores, keys, values, thr, frac, n_kept, return_indices=False, return_plan=False):
        out = real(scores, keys, values, thr, frac, n_kept, True, True)
        seen.append((scores.clone(), keys.clone(), values.clone(), thr, frac, n_kept, out))
        return out[0], out[1], out[2] if return_indices else None, *(out[3:] if return_plan else (None, None))

    monkeypatch.setattr(nat, "merging_compress", recording)
    return seen


def _presses():
    from kvpress_b200 import (ComposedPress, CriticalKVPress, ExpectedAttentionPress, KnormPress, MergingPress,
                              PrefillDecodingPress, PyramidKVPress, SnapKVPress)

    return {
        "knorm": lambda: MergingPress(KnormPress(0.5)),
        "snapkv": lambda: MergingPress(SnapKVPress(0.5, window_size=16), similarity_threshold=0.2),
        "expected": lambda: MergingPress(ExpectedAttentionPress(0.4), merge_fraction=0.75),
        "critical": lambda: MergingPress(CriticalKVPress(KnormPress(0.5))),
        "pyramid": lambda: MergingPress(PyramidKVPress(0.5, window_size=16)),
        "composed": lambda: ComposedPress([MergingPress(KnormPress(0.3)), KnormPress(0.2)]),
        "prefill_decoding": lambda: PrefillDecodingPress(prefilling_press=MergingPress(KnormPress(0.5))),
    }


@gpu
@pytest.mark.parametrize("name", ["knorm", "snapkv", "expected", "critical", "pyramid", "composed", "prefill_decoding"])
def test_press_on_a_tiny_llama(calls, name):
    model, cache = tiny_gpu_llama(), DynamicCache()
    ids = gpu_ids(240)
    with _presses()[name]()(model):
        model.model(input_ids=ids, past_key_values=cache)
    assert len(calls) == 2  # one merge per layer
    for layer, (scores, k, v, thr, frac, n_kept, (k_out, v_out, idx, target, sim)) in zip(cache.layers, calls):
        assert n_kept == int(k.shape[2] * 0.5) or name in ("expected", "composed")
        want = O.select_lowest_index_ties(scores.to(k.dtype).cpu(), n_kept).to(DEV)
        assert torch.equal(idx.long(), want) and torch.equal(k_out, O.gather_rows(k, want.long()))
        assert_plan(k, idx, target, sim)
        assert_values(v, idx, target, sim, thr, frac, v_out)
        if name != "composed":
            assert torch.equal(layer.keys, k_out) and torch.equal(layer.values, v_out)


@gpu
def test_press_merge_keeps_the_reference_contract():
    """merge(keys, values, indices): indices in any order, keys returned as they are, full-shape values with the merged
    rows at the kept positions and the evicted rows untouched."""
    from kvpress_b200 import KnormPress, MergingPress

    k, v = inputs(1, 2, 500, 64, torch.bfloat16, seed=37)
    kept = random_kept(1, 2, 500, 200, seed=37)
    shuffled = kept.gather(2, torch.rand(kept.shape, device=DEV).argsort(dim=-1)).long()
    press = MergingPress(KnormPress(0.6))
    keys, values = press.merge(k, v, shuffled)
    assert keys is k and values.shape == v.shape
    v_out = _native().merging_merge(k, v, kept, 0.0, 1.0)[0]
    assert torch.equal(values.gather(2, kept.long().unsqueeze(-1).expand(-1, -1, -1, 64)), v_out)
    ev = MB.complement(kept, 500).unsqueeze(-1).expand(-1, -1, -1, 64)
    assert torch.equal(values.gather(2, ev), v.gather(2, ev))
