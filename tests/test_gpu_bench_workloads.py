"""The calls bench.py times, checked the way bench.py runs them.

bench.py times CUDA-graph replays of `bench.run_native` (one `native.GraphedCall` per input set, replayed as
`calls[i % n]` with no synchronisation between steps), a 40-layer SnapKV pass captured into one graph, and the
host-buffer path of `host_staging.compress_host`. This file runs the same code on the same inputs:

1. Every `bench.WORKLOADS` entry at its exact shape, from `bench.make_inputs` with the bench's seeds and its L2-driven
   number of input sets (at least 2), replayed 2n times in bench order. Then, for every set:
     * the graph outputs equal an eager `bench.run_native` call on the same set, bitwise;
     * the kept positions, recovered from V' by exact row matching against V (the V rows of a head are asserted
       distinct first), are strictly ascending, n_kept per row, and K' is the exact gather of them (KeyRerotation:
       every K' element is one of the admissible re-rotated values);
     * the kept positions are the lowest-index-ties top-n_kept of the eager score call (StreamingLLM: the sinks and
       the most recent positions), and that score call is within the float64 bars of the scorer's sweep;
     * AdaKV(ExpectedAttention): the pruned flat index list equals one rebuilt from the eager scores with the canonical
       selection rule (safeguard, finfo.max, bottom H * (S - n_kept) of the flat scores), in its order.
   After that, replaying any one graph leaves every other graph's outputs unchanged, two back-to-back replays of one
   graph agree, and a replay after the inputs were overwritten in place equals a fresh eager call.
2. Capture, in-place update and replay of the entry points of the bench's workloads, in bf16 and fp16, at a small
   shape and at one with more select tiles than one wave of the persistent select kernel.
3. Several compress calls captured into one graph (the bench's multi-layer extra), keeping every layer's outputs or,
   as `prefill_pass` does, only the last layer's.
4. The host-buffer path in the mode bench.py picks (`zero_copy`, or `staged` for ExpectedAttention), one kv head per
   chunk, at the bench shapes.
Measured on an H100 80GB HBM3 (700 W power limit): the file runs in about 55 s, most of it the first test's CUDA and
cuBLAS start-up. There the SnapKV host path at 128k was not bitwise equal to the device call on the whole cache (its
softmax partials are split over CTAs by the row count), and the ExpectedAttention one was.
"""
import math
import sys
from pathlib import Path

import pytest
import torch

from oracle import press_oracle as O
from tests.gpu_support import (assert_e_small, assert_keydiff_vs_ref, assert_rerotated, assert_vs_ref64, ea_ref64,
                               _forced_head, _forced_tail, _gather, kd_chain, keydiff_error_bound, keydiff_ref64,
                               knorm_ref64, _name, _native, _same, snap_ref64)

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import bench  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = [torch.bfloat16, torch.float16]


def _n_kept(w: dict) -> int:
    return w.get("n_kept") or bench.kept_count(w["S"], bench.effective_ratio(w))


def _n_sets(w: dict) -> int:
    """bench.py's count of rotating input sets, but at least 2 so that every workload interleaves graphs."""
    bytes_per_set = 2 * w["B"] * w["Hkv"] * w["S"] * w["D"] * 2
    return max(2, min(8, math.ceil(4 * bench.L2_BYTES / bytes_per_set)))


def _all_same(a, b) -> bool:
    return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))


def _clone(outs):
    return tuple(None if t is None else t.clone() for t in outs)


# ---------------------------------------------------------------------------------------------------
# kept positions from V' alone
# ---------------------------------------------------------------------------------------------------
_HASH_W = torch.randint(-2 ** 62, 2 ** 62, (512,), generator=torch.Generator().manual_seed(5)) | 1


def _row_hash(x: torch.Tensor) -> torch.Tensor:
    """[N, D] 16-bit rows -> int64 [N]: a random linear form of the bit patterns (mod 2^64). Equal rows hash equal, so
    distinct hashes prove distinct rows."""
    bits = x.contiguous().view(torch.int16).to(torch.int64) & 0xFFFF
    return (bits * _HASH_W[:x.shape[-1]].to(x.device)).sum(-1)


def kept_positions(v: torch.Tensor, v_out: torch.Tensor) -> torch.Tensor:
    """int64 [B, H, n]: the position in V of every row of V', by exact row matching; asserts that the V rows of every
    head are distinct (so the match is unique) and that every V' row is a V row at that position, bitwise."""
    B, H, S, _ = v.shape
    pos = torch.empty(v_out.shape[:3], dtype=torch.int64, device=v.device)
    for b in range(B):
        for h in range(H):
            hv, order = _row_hash(v[b, h]).sort()
            assert bool((hv[1:] != hv[:-1]).all()), f"V rows of head ({b}, {h}) are not distinct"
            hk = _row_hash(v_out[b, h])
            i = torch.searchsorted(hv, hk).clamp_max(S - 1)
            assert bool((hv[i] == hk).all()), f"a V' row of head ({b}, {h}) is no row of V"
            pos[b, h] = order[i]
    assert _same(v_out, _gather(v, pos)), "V' rows do not match V rows exactly"
    return pos


# ---------------------------------------------------------------------------------------------------
# 1. every bench workload, replayed as the bench replays it
# ---------------------------------------------------------------------------------------------------
def _check_kept(w, k, v, n_kept, out, what):
    """positions of V' (strictly ascending, n_kept per row) and, unless K' is re-rotated, K' = K[pos]"""
    k_out, v_out = out
    pos = kept_positions(v, v_out)
    assert pos.shape == (w["B"], w["Hkv"], n_kept), what
    assert bool((pos[..., 1:] > pos[..., :-1]).all()), f"{what}: kept positions are not strictly ascending"
    if w["scorer"] != "knorm_rerotate":
        assert _same(k_out, _gather(k, pos)), f"{what}: K' is not K at the kept positions"
    return pos


def _check_selection(pos, scores, n_kept, what):
    want = O.select_lowest_index_ties(scores.cpu(), n_kept)
    assert torch.equal(pos.cpu(), want), f"{what}: not the lowest-index-ties top-{n_kept} of the eager scores"


def check_expected_attention(w, k, v, extra, n_kept, out, what):
    S = w["S"]
    pos = _check_kept(w, k, v, n_kept, out, what)
    sc = _native().expected_attention_score(k, v, extra["mu"], extra["cov"], 0.0, 4, True)
    assert_vs_ref64(sc, ea_ref64(k, v, extra["mu"], extra["cov"], 0.0, 4, True), _forced_head(S, 4), what)
    _check_selection(pos, sc, n_kept, what)


def check_snapkv(w, k, v, extra, n_kept, out, what):
    S, q = w["S"], extra["q_window"]
    pos = _check_kept(w, k, v, n_kept, out, what)
    sc = _native().snapkv_score(k, q, 64, 5)
    G = q.shape[1] // k.shape[1]
    # one kv head at a time: at Hq = 64 a head's 512 x S float64 logits are 512 MiB
    ref = torch.cat([snap_ref64(q[:, h * G:(h + 1) * G], k[:, h:h + 1], 64, 5) for h in range(k.shape[1])], dim=1)
    assert_vs_ref64(sc, ref, _forced_tail(S, 64), what, ftz=True)
    _check_selection(pos, sc, n_kept, what)


def check_knorm(w, k, v, extra, n_kept, out, what):
    pos = _check_kept(w, k, v, n_kept, out, what)
    # the scores of the compress call itself: the cluster path (decoding_knorm) has no separate score kernel
    sc = _native().knorm_compress(k, v, n_kept, return_scores=True)[3]
    assert_vs_ref64(sc, knorm_ref64(k), torch.zeros(w["S"], dtype=torch.bool), what)
    _check_selection(pos, sc, n_kept, what)


def check_knorm_rerotate(w, k, v, extra, n_kept, out, what):
    pos = _check_kept(w, k, v, n_kept, out, what)
    sc = _native().knorm_score(k)
    assert_vs_ref64(sc, knorm_ref64(k), torch.zeros(w["S"], dtype=torch.bool), what)
    assert_rerotated(k, v, sc, n_kept, extra["inv_freq"], (out[0], out[1], pos), what)


def check_keydiff(w, k, v, extra, n_kept, out, what):
    pos = _check_kept(w, k, v, n_kept, out, what)
    sc = _native().keydiff_score(k)
    ref = keydiff_ref64(k)
    E = keydiff_error_bound(k, kd_chain(w["S"], w["D"]))
    assert_e_small(E, ref, what)
    assert_keydiff_vs_ref(sc, ref, E, what)
    _check_selection(pos, sc, n_kept, what)


def check_streaming(w, k, v, extra, n_kept, out, what):
    pos = _check_kept(w, k, v, n_kept, out, what)
    assert torch.equal(pos.cpu(), O.streaming_kept(w["S"], n_kept, 4).expand_as(pos.cpu())), what


def check_adakv_ea(w, k, v, extra, n_kept, out, what):
    """The pruned flat index list rebuilt from the eager scores: the n_kept / 5 best of every head are safeguarded
    (finfo.max), then the H * (S - n_kept) lowest of the flat [B, H * S] scores are pruned, ties to the lowest index."""
    B, H, S = w["B"], w["Hkv"], w["S"]
    assert out[1] is None
    sc = _native().expected_attention_score(k, v, extra["mu"], extra["cov"], 1e-2, 4, True)
    assert_vs_ref64(sc, ea_ref64(k, v, extra["mu"], extra["cov"], 1e-2, 4, True), _forced_head(S, 4), what)
    sc = sc.cpu()
    safe = O.select_lowest_index_ties(sc, int(n_kept * 0.2))
    sc = sc.scatter(-1, safe, torch.finfo(sc.dtype).max)
    want = O.select_lowest_index_ties((-sc).reshape(B, 1, H * S), H * (S - n_kept))
    got = out[0].long().cpu()
    assert got.shape == want.shape, what
    bad = got != want
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} of {got.numel()} pruned indices differ from the canonical list"


CHECKERS = {
    "expected_attention": check_expected_attention,
    "snapkv": check_snapkv,
    "knorm": check_knorm,
    "knorm_rerotate": check_knorm_rerotate,
    "keydiff": check_keydiff,
    "streaming": check_streaming,
    "adakv_ea": check_adakv_ea,
}


def test_every_bench_workload_has_a_checker():
    missing = sorted({w["scorer"] for w in bench.WORKLOADS.values()} - set(CHECKERS))
    assert not missing, f"bench workloads with no checker: {missing}"


def _overwrite(inputs, new):
    """Copies the tensors of `new` into `inputs` in place: (K, V, extra) of bench.make_inputs."""
    for a, b in zip(inputs[:2], new[:2]):
        a.copy_(b)
    for name, t in inputs[2].items():
        t.copy_(new[2][name])


@pytest.mark.parametrize("name", list(bench.WORKLOADS))
def test_bench_workload_replayed(name):
    nat = _native()
    w = bench.WORKLOADS[name]
    n_kept = _n_kept(w)
    n = _n_sets(w)
    sets = [bench.make_inputs(w, DEV, bench.rank_seed(0, i)) for i in range(n)]
    graphs = [nat.capture(lambda s=s: bench.run_native(w, s[0], s[1], s[2], n_kept)) for s in sets]
    for i in range(2 * n):  # bench.timed_loop: calls[i % n], no synchronisation between steps
        graphs[i % n].replay()
    torch.cuda.synchronize()
    got = [_clone(g.outputs) for g in graphs]

    for i, (k, v, extra) in enumerate(sets):
        what = f"{name} set {i}"
        assert _all_same(got[i], bench.run_native(w, k, v, extra, n_kept)), f"{what}: graph replay != eager call"
        CHECKERS[w["scorer"]](w, k, v, extra, n_kept, got[i], what)

    # one graph's replay leaves every other graph's outputs alone (no two private pools alias)
    for j in range(n):
        graphs[j].replay()
        torch.cuda.synchronize()
        for i in range(n):
            assert _all_same(graphs[i].outputs, got[i]), f"{name}: replaying graph {j} changed graph {i}'s outputs"
    # the per-call memset re-zeroes counters, histograms and flags on every replay
    first = _clone(graphs[0].replay())
    second = graphs[0].replay()
    torch.cuda.synchronize()
    assert _all_same(first, second), f"{name}: two back-to-back replays differ"
    # the graph reads its inputs at replay time
    _overwrite(sets[0], bench.make_inputs(w, DEV, bench.rank_seed(0, 999)))
    replayed = _clone(graphs[0].replay())
    torch.cuda.synchronize()
    k, v, extra = sets[0]
    assert _all_same(replayed, bench.run_native(w, k, v, extra, n_kept)), f"{name}: replay on new inputs != eager"
    assert not _same(replayed[0], got[0][0]), f"{name}: the replay did not see the new inputs"


# ---------------------------------------------------------------------------------------------------
# 2. capture / in-place update / replay of every entry point the bench calls
# ---------------------------------------------------------------------------------------------------
ENTRIES = ["ea_cov_vnorm", "ea_cov_novnorm", "ea_nocov_vnorm", "ea_nocov_novnorm", "snapkv", "streaming",
           "scores_compress", "scores_select", "scores_compress_rerotate"]
# (B, H, S): R = 4 rows of about 3000 positions; and R * ceil(S / 256) select tiles above one wave of the persistent
# select kernel (SMs x 8 CTAs of 256 threads at most)
SHAPES = {"small": (2, 2, 3000), "over_a_wave": (2, 4, 40000)}
ENTRY_G, ENTRY_D, ENTRY_W = 4, 128, 64


def entry_inputs(entry, dtype, B, H, S, seed) -> dict:
    gen = torch.Generator(device=DEV).manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=gen, device=DEV)  # noqa: E731
    G, D = ENTRY_G, ENTRY_D
    t = {"k": rn(B, H, S, D).to(dtype), "v": rn(B, H, S, D).to(dtype)}
    if entry.startswith("ea"):
        t["mu"] = (0.5 * rn(B, H * G, D)).to(dtype)
        if "_cov" in entry:
            a = rn(B, H * G, D, D) / D ** 0.5
            t["cov"] = (a @ a.transpose(-1, -2)).to(dtype)
    if entry == "snapkv":
        t["q"] = (1.5 * rn(B, H * G, ENTRY_W, D)).to(dtype)
    if entry.startswith("scores"):
        t["sc"] = rn(B, H, S).to(dtype)
    if entry == "scores_compress_rerotate":
        theta = 10000.0 + 490000.0 * float(torch.rand((), generator=gen, device=DEV))
        t["inv_freq"] = (1.0 / (theta ** (torch.arange(0, D, 2, device=DEV).float() / D))).contiguous()
    return t


def entry_call(entry, t, n_kept):
    """the entry point's score call (where it has one) and its compress / select call, indices and scores returned"""
    nat = _native()
    k, v = t["k"], t["v"]
    if entry.startswith("ea"):
        vn = entry.endswith("_vnorm")
        eps = 1e-2 if vn else 0.0
        cov = t.get("cov")
        return (nat.expected_attention_score(k, v, t["mu"], cov, eps, 4, vn),
                *nat.expected_attention_compress(k, v, t["mu"], cov, eps, 4, vn, n_kept, return_indices=True,
                                                 return_scores=True))
    if entry == "snapkv":
        return (nat.snapkv_score(k, t["q"], ENTRY_W, 5),
                *nat.snapkv_compress(k, v, t["q"], ENTRY_W, 5, n_kept, return_indices=True, return_scores=True))
    if entry == "streaming":
        return nat.streaming_compress(k, v, n_kept, 4, return_indices=True)
    if entry == "scores_compress":
        return nat.scores_compress(t["sc"], k, v, n_kept, return_indices=True)
    if entry == "scores_select":
        return (nat.scores_select(t["sc"], n_kept),)
    return nat.scores_compress_rerotate(t["sc"], k, v, n_kept, t["inv_freq"], return_indices=True)


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("entry", ENTRIES)
def test_entry_point_replays_under_capture(entry, dtype, shape):
    nat = _native()
    B, H, S = SHAPES[shape]
    if shape == "over_a_wave":
        props = torch.cuda.get_device_properties(0)
        assert B * H * -(-S // 256) > props.multi_processor_count * (props.max_threads_per_multi_processor // 256)
    n_kept = O.kept_count(S, 0.5)
    seed = 100 * ENTRIES.index(entry) + 10 * DTYPES.index(dtype) + list(SHAPES).index(shape)
    t = entry_inputs(entry, dtype, B, H, S, seed)
    what = f"{entry} {_name(dtype)} {shape}"
    eager = _clone(entry_call(entry, t, n_kept))
    g = nat.capture(lambda: entry_call(entry, t, n_kept))
    # the first replay runs on a workspace fresh from the graph's pool; the second finds the first one's counters
    assert _all_same(g.replay(), eager), f"{what}: first graph replay != eager call"
    for name, x in entry_inputs(entry, dtype, B, H, S, seed + 50000).items():  # inputs updated in place
        t[name].copy_(x)
    out = _clone(g.replay())
    torch.cuda.synchronize()
    fresh = entry_call(entry, t, n_kept)
    assert _all_same(out, fresh), f"{what}: graph replay != eager call on the new inputs"
    assert not _all_same(out, eager), f"{what}: the replay did not see the new inputs"


# ---------------------------------------------------------------------------------------------------
# 3. several layers' compress calls in one graph
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("keep", ["every_layer", "last_layer"])
@pytest.mark.parametrize("name", ["snapkv_128k_70b", "ea_128k"])
def test_layers_captured_into_one_graph(name, keep):
    """bench.extra_layer_split captures a whole prefill pass into one graph, and its `prefill_pass` drops every
    layer's outputs: inside the capture a layer's outputs and workspace go back to the graph's pool for the next."""
    nat = _native()
    w = bench.WORKLOADS[name]
    n_kept = _n_kept(w)
    layers = [bench.make_inputs(w, DEV, bench.rank_seed(0, 100 + i)) for i in range(4)]

    def every_layer():
        return [bench.run_native(w, k, v, extra, n_kept) for k, v, extra in layers]

    def last_layer():  # like prefill_pass, but the last layer's outputs are returned
        out = None
        for k, v, extra in layers:
            out = bench.run_native(w, k, v, extra, n_kept)
        return [out]

    g = nat.capture(every_layer if keep == "every_layer" else last_layer)
    g.replay()
    g.replay()
    torch.cuda.synchronize()
    kept = layers if keep == "every_layer" else layers[-1:]
    assert len(g.outputs) == len(kept)
    for i, (out, (k, v, extra)) in enumerate(zip(g.outputs, kept)):
        assert _all_same(out, bench.run_native(w, k, v, extra, n_kept)), f"{name} {keep}: output {i} != eager call"


# ---------------------------------------------------------------------------------------------------
# 4. the host-buffer path in the mode bench.py picks
# ---------------------------------------------------------------------------------------------------
HOST_MODES = {"knorm_128k": "zero_copy", "keydiff_128k": "zero_copy", "snapkv_128k_70b": "zero_copy",
              "streaming_128k": "zero_copy", "ea_128k": "staged"}


@pytest.mark.parametrize("name", list(HOST_MODES))
def test_host_path_in_bench_mode(name):
    """Pinned host K/V through compress_host with one kv head per chunk equal the device path, bitwise. Knorm, KeyDiff
    and StreamingLLM score every position on its own or from per-row sums in a fixed order, so the device call on the
    whole cache is the reference. ExpectedAttention and SnapKV split each row's softmax over CTAs by the number of rows
    of the call, so the reference is the device call on one kv head, which is what a chunk runs."""
    from kvpress_b200 import host_staging
    _native()
    w = bench.WORKLOADS[name]
    n_kept = _n_kept(w)
    mode = HOST_MODES[name]
    kh, vh, extra = bench.make_inputs(w, DEV, bench.rank_seed(0, 99), pinned_host=True)
    assert kh.is_pinned() and vh.is_pinned()
    params = dict(extra)
    if w["scorer"] == "snapkv":
        params.update(window=64, kernel_size=5)
    if w["scorer"] == "expected_attention":
        params.update(epsilon=0.0, n_sink=4, use_vnorm=True)
    k2, v2 = host_staging.compress_host(w["scorer"], kh, vh, n_kept, device=DEV, heads_per_chunk=1,
                                        values_zero_copy=(mode == "zero_copy"), **params)
    assert k2.is_pinned() and v2.is_pinned()
    kd, vd = kh.to(DEV), vh.to(DEV)
    if w["scorer"] in ("knorm", "keydiff", "streaming"):
        k_ref, v_ref = bench.run_native(w, kd, vd, extra, n_kept)
        assert _same(k2, k_ref.cpu()) and _same(v2, v_ref.cpu()), f"{name} {mode}: host path != device path"
        return
    G = w["Hq"] // w["Hkv"]
    for h in range(w["Hkv"]):
        one = {key: t[:, h * G:(h + 1) * G] for key, t in extra.items()}
        k_ref, v_ref = bench.run_native(w, kd[:, h:h + 1], vd[:, h:h + 1], one, n_kept)
        assert _same(k2[:, h:h + 1], k_ref.cpu()) and _same(v2[:, h:h + 1], v_ref.cpu()), \
            f"{name} {mode}: kv head {h} of the host path != the device call on that head"
    whole = bench.run_native(w, kd, vd, extra, n_kept)
    print(f"[measured] {name}: host path bitwise equal to the device call on the whole cache: "
          f"{_same(k2, whole[0].cpu()) and _same(v2, whole[1].cpu())}")
