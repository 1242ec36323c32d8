"""The shared selection and compaction stages against an exact reference: every 16-bit key, every head_dim, rows past the
persistent grid, strided K / V.

Every press ends in the same two stages. The score stage writes each row's ordered 16-bit keys (`ordered_key16`,
common.cuh) and the 256-bin histogram of their high bytes; caller-supplied scores get theirs from
`keys_from_scores_kernel` (knorm.cu). `select_compact_kernel` (select_compact.cu) then finds each row's top n_kept and
copies the kept K / V rows; `streaming_compact_kernel` copies StreamingLLM's closed-form ranges. Unlike scoring, this stage
has an exact contract (DESIGN.md §2): keep the n_kept largest scores in the cache dtype, ties to the lowest position,
-0 == +0, NaN (either sign, any payload) above +inf, rows in position order. So every bar here is exact:
  * `idx` is int32 and equal to the canonical selection: `oracle.press_oracle.select_lowest_index_ties` of the same 16-bit
    scores. A row's canonical order (the oracle's key, stable descending sort) is computed once and `sort(order[:n])` is
    taken for each n_kept; each case also checks one n_kept against the oracle itself;
  * `scores_select`, `scores_compress` and `scores_compress_rerotate` return that same idx;
  * K' and V' are bitwise gathers (K / V hold random bit patterns, NaN payloads included); the re-rotated K' is one of the
    results the admissible-set helper of tests/test_gpu_keydiff_rerotation_sweep.py allows;
  * no bounded wait expired (`native.workspace_check` after every call; after the last one where calls are enqueued
    back to back or on two streams at once).
Before each call the outputs' blocks are poisoned: blocks of the outputs' sizes are allocated in the order the binding
allocates its outputs, filled with 0xFF and freed, and the test asserts that the outputs landed on them. An element the
kernels never write reads 0xFFFF (a NaN; idx -1), never a stale value of an earlier call.

The cases: (1) rows holding all 65536 bit patterns of a dtype (and each pattern 3x, spread over tiles), with n_kept at
every high-byte bin boundary and +-1, and at every low-byte boundary of the NaN, +inf, -inf, zero and subnormal bins;
(2) planted threshold ties on negative and mixed-sign scores, straddling a tile and a refine group, only in the first or
the last (padded) tile, in the lowest populated bin, in the NaN bin and at low bytes 0x00 / 0xFF; all-NaN, all -inf and
mixed +-0 rows; (3) S on both sides of 1, 16 and 17 tiles (one and two refine groups) up to a flat 8 x 128k AdaKV row and a
4M-position select row, B·H up to 65535, work-item counts from 2 to past 64 per SM; (4) every head_dim 8..256 with one
tile's kept count on both sides of the copy loop's batch edges, through five K / V layouts, and StreamingLLM over the
same grid; (5) the entry-point contracts: fp32 scores, score strides, graph replay, growing / shrinking shapes on one
stream, two streams. CPU tests check `ordered_key16` itself (compiled for the host) against the oracle's order, and that
the boundary lists here are derived from the constants the sources use.

On an H100 80GB HBM3 (700 W power limit) the 238 GPU cases pass in about 100 s. No case found a kernel bug.
"""
import ctypes
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import press_oracle as O
from tests.gpu_support import (INF_BITS, TILE, TILE_THREADS, _bits, _kv_out_bytes, _landed, _name, _native, _poison,
                               _score_copy_bytes, _sm_count, all_patterns, assert_gather, assert_idx,
                               canonical, canonical_order, copy_edges, edge_counts, key16, kv_for, mixed_scores,
                               key_space_n_kept, oracle_key, rand_bits, rerotation_admissible, rope_inv_freq,
                               threshold_patterns, _pattern_keys)

gpu = pytest.mark.gpu
DEV = "cuda:0"
CSRC = Path(__file__).resolve().parent.parent / "kvpress_b200" / "csrc"
DTYPES = [torch.bfloat16, torch.float16]

# the constants of common.cuh / select_compact.cu the boundary lists are derived from (checked by a CPU test)
SFX_STRIDE = 264    # kSfxStride
TILES_PER_WARP = 2  # kTilesPerWarp
GROUP_TILES = TILE_THREADS // 32 * TILES_PER_WARP  # kGroupTiles: tiles per refine item
SEL_U = 3           # kSelU: 16-byte vectors per thread and batch in copy_rows_kv of the compact items
SEL_CTAS = 3        # kSelCtas
REROT_CTAS = 4      # kRerotCtas
STREAM_U = 4        # copy_rows_kv<4> of streaming_compact_kernel
MAX_ROWS = 65535    # B·Hkv: gridDim.y of the score kernels


SHAPE_TILES = (1, GROUP_TILES, GROUP_TILES + 1, 2 * GROUP_TILES, 2 * GROUP_TILES + 1)
SHAPE_S = [1, 2] + [t * TILE + d for t in SHAPE_TILES for d in (-1, 0, 1)]
HEAD_DIMS = list(range(8, 257, 8))
LAYOUTS = ["contiguous", "k_contiguous_v_bshd", "v_row_slice", "k_broadcast_head", "offset_views"]


# ---------------------------------------------------------------------------------------------------
# calls: poisoned outputs (tests/gpu_support.py _poison), workspace check
# ---------------------------------------------------------------------------------------------------
def _select_problem(nat, scores, n):
    B, H, S = scores.shape
    p = nat.KvpProblem()
    p.B, p.Hkv, p.Hq, p.S, p.D, p.n_kept, p.dtype = B, H, H, S, 8, int(n), nat._DTYPES[scores.dtype]
    return p


def _check_ws(nat, p, scorer=None):
    scorer = nat.SCORER_GENERIC if scorer is None else scorer
    nat.workspace_check(p, scorer, nat._workspace(p, scorer, torch.device(DEV)))


def call_select(nat, scores, n, check=True):
    """`check`: workspace_check after the call (it synchronises the stream)"""
    B, H, _ = scores.shape
    ptrs = _poison(_score_copy_bytes(scores, scores.dtype), B * H * n * 4)
    idx = nat.scores_select(scores, n)
    _landed(ptrs, idx)
    if n and check:
        _check_ws(nat, _select_problem(nat, scores, n))
    return idx


def call_compress(nat, scores, k, v, n, inv=None, check=True):
    ptrs = _poison(_score_copy_bytes(scores, k.dtype), *_kv_out_bytes(k, n))
    if inv is None:
        out = nat.scores_compress(scores, k, v, n, return_indices=True)
    else:
        out = nat.scores_compress_rerotate(scores, k, v, n, inv, return_indices=True)
    _landed(ptrs, *out)
    if n and check:
        _check_ws(nat, nat.make_problem(k, v, n))
    return out


def call_streaming(nat, k, v, n, n_sink):
    ptrs = _poison(*_kv_out_bytes(k, n))
    out = nat.streaming_compress(k, v, n, n_sink, return_indices=True)
    _landed(ptrs, *out)
    return out


def assert_rerotated(k_out, k, want, inv, what):
    adm = _bits(rerotation_admissible(k, want, inv))
    hit = (adm == _bits(k_out)[None]).any(0)
    assert hit.all(), f"{what}: {int((~hit).sum())} of {hit.numel()} re-rotated K' elements not admissible"


def check_entry_points(scores, k, v, kr, ns, what, order=None, inv=None):
    """Every n_kept of `ns` through scores_select, scores_compress (K / V) and scores_compress_rerotate (kr / V, when
    `inv` is given): the canonical idx from all three, bitwise gathers, admissible re-rotated keys."""
    nat = _native()
    order = canonical_order(scores) if order is None else order
    n0 = ns[len(ns) // 2]  # the shortcut through the canonical order is the oracle's selection
    assert torch.equal(canonical(order, n0).cpu(), O.select_lowest_index_ties(scores.cpu(), n0)), what
    for n in ns:
        w = f"{what} n_kept={n}"
        want = canonical(order, n)
        assert_idx(call_select(nat, scores, n), want, w + " scores_select")
        k_out, v_out, idx = call_compress(nat, scores, k, v, n)
        assert_idx(idx, want, w + " scores_compress")
        assert_gather(k_out, k, want, w + " K'")
        assert_gather(v_out, v, want, w + " V'")
        if inv is not None:
            k_out, v_out, idx = call_compress(nat, scores, kr, v, n, inv)
            assert_idx(idx, want, w + " scores_compress_rerotate")
            assert_gather(v_out, v, want, w + " rerotate V'")
            assert_rerotated(k_out, kr, want, inv, w + " rerotate")


def n_kept_values(S: int):
    return sorted({n for n in (1, 2, S // 2, S - 1, S) if 1 <= n <= S})


# ---------------------------------------------------------------------------------------------------
# CPU: ordered_key16 against the oracle's order; the boundary lists follow the sources' constants
# ---------------------------------------------------------------------------------------------------
_KEY_PROGRAM = r"""
#include <stdio.h>
#include "common.cuh"
int main() {
    static uint16_t out[2][65536];
    for (unsigned b = 0; b < 65536u; ++b) {
        out[0][b] = kvp::ordered_key16((uint16_t)b, 0x7F80u);  // bf16
        out[1][b] = kvp::ordered_key16((uint16_t)b, 0x7C00u);  // fp16
    }
    fwrite(out, sizeof(out), 1, stdout);
    return 0;
}
"""


def _nvcc():
    from kvpress_b200 import build
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        return None
    return nvcc if Path(nvcc).is_absolute() and Path(nvcc).exists() else shutil.which(nvcc)


def test_ordered_key16_is_the_oracle_order(tmp_path):
    """`ordered_key16` of all 65536 patterns of each dtype, compiled for the host from common.cuh: sorting a seeded
    permutation of them by key gives the oracle's order, with equal keys exactly where the oracle ties."""
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = tmp_path / "keys.cu"
    src.write_text(_KEY_PROGRAM)
    exe = tmp_path / "keys"
    subprocess.run([nvcc, "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-I", str(CSRC), str(src),
                    "-o", str(exe)], check=True, capture_output=True)
    keys = np.frombuffer(subprocess.run([str(exe)], check=True, capture_output=True).stdout, dtype=np.uint16)
    keys = torch.from_numpy(keys.astype(np.int64)).view(2, 65536)
    for i, dtype in enumerate(DTYPES):
        pats = all_patterns(dtype)
        perm = torch.randperm(65536, generator=torch.Generator().manual_seed(i))
        row = pats[perm]
        k = keys[i][(row.view(torch.int16).long() + 65536) % 65536]
        ref = canonical_order(row[None])[0]
        assert torch.equal(canonical(ref, 1000), O.select_lowest_index_ties(row[None, None], 1000)[0, 0])
        got = torch.sort(k, descending=True, stable=True).indices
        assert torch.equal(got, ref), f"{_name(dtype)}: the key order is not the oracle's"
        ok = oracle_key(row)[ref]
        assert torch.equal(k[ref][1:] == k[ref][:-1], ok[1:] == ok[:-1]), f"{_name(dtype)}: key ties differ from the oracle's"
        # what the order means: NaN of either sign on top, then +inf; -inf last; -0 and +0 one key
        nan = torch.isnan(row.float())
        assert int(nan.sum()) == 2 * (0x7FFF - INF_BITS[dtype]) and (k[nan] == 0xFFFF).all()
        assert int(k[~nan].max()) == int(k[row == float("inf")]) and int(k.min()) == int(k[row == float("-inf")])
        zeros = k[row == 0]
        assert zeros.numel() == 2 and zeros[0] == zeros[1]
        # and the restatement the GPU cases place their bin edges with is this function
        assert torch.equal(keys[i], key16(torch.arange(65536), dtype)), f"{_name(dtype)}: restated key differs"


def _constant(text: str, name: str) -> int:
    m = re.search(rf"(?:constexpr\s+\w+\s+{name}\s*=\s*|#define\s+{name}\s+)(\w+)", text)
    assert m, name
    return int(m.group(1), 0)


def test_boundaries_follow_the_source_constexprs():
    """The constants the boundary lists are derived from are the sources'; the lists hold every edge they imply."""
    common = (CSRC / "common.cuh").read_text()
    sc = (CSRC / "select_compact.cu").read_text()
    assert _constant(common, "kTile") == TILE and _constant(common, "kTileThreads") == TILE_THREADS
    assert _constant(common, "kSfxStride") == SFX_STRIDE and SFX_STRIDE >= TILE + 2
    assert _constant(sc, "kTilesPerWarp") == TILES_PER_WARP
    assert "kGroupTiles = (kTileThreads / 32) * kTilesPerWarp" in sc
    assert _constant(sc, "kSelU") == SEL_U and _constant(sc, "kSelCtas") == SEL_CTAS
    assert _constant(sc, "kRerotCtas") == REROT_CTAS
    assert "copy_rows_kv<kSelU>(" in sc
    copy = re.search(r"void copy_rows_kv\(.*?\n}", sc, re.S).group(0)
    assert "base += 2 * STEP" in copy  # two steps per loop iteration, as copy_edges assumes
    streaming = re.search(r"streaming_compact_kernel\(.*?\n}", sc, re.S).group(0)
    assert re.findall(r"copy_rows_kv<(\d+)>", streaming) == [str(STREAM_U)]
    assert "p->B * p->Hkv > 65535" in (CSRC / "api.cu").read_text() and MAX_ROWS == 65535
    # S on both sides of 1, one group, one group + 1, two groups and two groups + 1 tiles
    for t in (1, GROUP_TILES, GROUP_TILES + 1, 2 * GROUP_TILES, 2 * GROUP_TILES + 1):
        assert {t * TILE - 1, t * TILE, t * TILE + 1} <= set(SHAPE_S)
    assert {1, 2} <= set(SHAPE_S)
    # head_dims: every vector count a row can have, and per D the counts on both sides of every copy edge
    assert [D // 8 for D in HEAD_DIMS] == list(range(1, 33))
    for u in (SEL_U, STREAM_U):
        step, double = copy_edges(u)
        assert (step, double) == (TILE_THREADS * u, 2 * TILE_THREADS * u)
        for nvec in range(1, 33):
            cs = edge_counts(nvec, u)
            for e in (step, double):
                below, at = (e - 1) // nvec, -(-e // nvec)
                if at + 1 <= TILE:  # reachable in one tile: the edge is straddled
                    assert below in cs and at in cs and e // nvec + 1 in cs
                    assert below * nvec < e <= at * nvec
    assert edge_counts(1, SEL_U) == [1, TILE]  # one vector per row never reaches a copy edge
    assert 767 // 3 in edge_counts(3, SEL_U) and 768 // 3 in edge_counts(3, SEL_U)


def test_reference_shortcut_is_the_oracle():
    """canonical(order, n) == O.select_lowest_index_ties at every n of rows full of ties and special values"""
    gen = torch.Generator().manual_seed(3)
    for dtype in DTYPES:
        pats = all_patterns(dtype)
        row = pats[torch.randint(0, 65536, (2, 3, 700), generator=gen)]
        row[..., ::3] = torch.tensor([0.0, -0.0, float("nan"), float("-inf")], dtype=dtype)[
            torch.randint(0, 4, (2, 3, 234), generator=gen)]
        order = canonical_order(row)
        for n in range(0, 701, 7):
            assert torch.equal(canonical(order, n), O.select_lowest_index_ties(row, n)), (dtype, n)


# ---------------------------------------------------------------------------------------------------
# 1. the whole key space
# ---------------------------------------------------------------------------------------------------


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("repeat", [1, 3], ids=["each_once", "each_thrice"])
def test_key_space(dtype, repeat):
    """Two rows, each all 65536 patterns (`repeat` times) in a seeded permutation: threshold ties straddle tiles."""
    gen = torch.Generator(device=DEV).manual_seed(10 + repeat)
    pats = all_patterns(dtype).to(DEV).repeat(repeat)
    S = pats.numel()
    perm = torch.stack([torch.randperm(S, generator=gen, device=DEV) for _ in range(2)])
    scores = pats[perm].view(1, 2, S)
    k, v, kr = kv_for(1, 2, S, 16, dtype, gen)
    inv = rope_inv_freq("theta1e4", 16).to(DEV)
    ns = key_space_n_kept(key16(pats.view(torch.int16).cpu(), dtype), dtype)
    check_entry_points(scores, k, v, kr, ns, f"key space {_name(dtype)} x{repeat}", inv=inv)


# ---------------------------------------------------------------------------------------------------
# 2. planted threshold ties
# ---------------------------------------------------------------------------------------------------
PLANT_S = 3 * GROUP_TILES * TILE - 77  # 3 refine groups, the last partial; the last tile padded
THRESHOLDS = ["neg_inf", "most_negative", "nan", "key_lo00", "key_loff", "zero_mixed_sign"]
PLACEMENTS = ["straddle_tile_and_group", "first_tile_only", "last_tile_only"]
PLANTED = [(t, p, dt) for t in THRESHOLDS for p in PLACEMENTS for dt in DTYPES]


def planted_row(kind, placement, dtype, gen, n_t=40):
    """One row: n_t positions hold the threshold key; the others are strictly above or below it (n_gt above)."""
    S = PLANT_S
    pats, keys = _pattern_keys(dtype)
    tie_pats = threshold_patterns(kind, dtype)
    T = int(key16(tie_pats[:1], dtype))
    above, below = pats[keys > T], pats[keys < T]
    if placement == "straddle_tile_and_group":
        g = GROUP_TILES * TILE
        tie_pos = torch.cat([torch.arange(5 * TILE - n_t // 4, 5 * TILE + n_t // 4),
                             torch.arange(g - n_t // 4, g + n_t // 4)])
    elif placement == "first_tile_only":
        tie_pos = torch.randperm(TILE, generator=gen)[:n_t]
    else:
        last = (S - 1) // TILE * TILE
        tie_pos = last + torch.randperm(S - last, generator=gen)[:n_t]
    n_t = tie_pos.numel()
    rest = torch.ones(S, dtype=torch.bool)
    rest[tie_pos] = False
    rest = rest.nonzero()[:, 0]
    rest = rest[torch.randperm(rest.numel(), generator=gen)]
    if above.numel() == 0:  # NaN: nothing ranks above it
        n_gt = 0
    elif below.numel() == 0:  # -inf: nothing ranks below it
        n_gt = rest.numel()
    else:
        n_gt = rest.numel() // 2
    row = torch.empty(S, dtype=torch.int16)
    row[tie_pos] = tie_pats[torch.randint(0, tie_pats.numel(), (n_t,), generator=gen)]
    if n_gt:
        row[rest[:n_gt]] = above[torch.randint(0, above.numel(), (n_gt,), generator=gen)]
    if rest.numel() > n_gt:
        row[rest[n_gt:]] = below[torch.randint(0, below.numel(), (rest.numel() - n_gt,), generator=gen)]
    return row, n_gt, n_t


@gpu
@pytest.mark.parametrize("kind,placement,dtype", PLANTED, ids=[f"{k}-{p}-{_name(dt)}" for k, p, dt in PLANTED])
def test_planted_threshold_ties(kind, placement, dtype):
    """n_kept takes exactly one tie, half, all but one and all of them; rows differ, n_gt is the same in each"""
    gen = torch.Generator().manual_seed(7 + 10 * THRESHOLDS.index(kind) + PLACEMENTS.index(placement))
    rows = [planted_row(kind, placement, dtype, gen) for _ in range(4)]
    n_gt, n_t = rows[0][1], rows[0][2]
    assert all(r[1] == n_gt and r[2] == n_t for r in rows)
    scores = torch.stack([r[0] for r in rows]).view(dtype).view(2, 2, PLANT_S).to(DEV)
    keys = key16(scores.view(torch.int16), dtype)
    T = int(key16(threshold_patterns(kind, dtype)[:1], dtype))
    assert ((keys > T).sum(-1) == n_gt).all() and ((keys == T).sum(-1) == n_t).all()
    if kind in ("nan", "zero_mixed_sign"):  # both signs among the ties
        tie_bits = scores.view(torch.int16)[keys == T]
        assert (tie_bits < 0).any() and (tie_bits >= 0).any()
    gen_d = torch.Generator(device=DEV).manual_seed(11)
    k, v, kr = kv_for(2, 2, PLANT_S, 64, dtype, gen_d)
    inv = rope_inv_freq("theta5e5", 64).to(DEV)
    ns = sorted({n for n in (n_gt + 1, n_gt + n_t // 2, n_gt + n_t - 1, n_gt + n_t) if 1 <= n <= PLANT_S})
    check_entry_points(scores, k, v, kr, ns, f"planted {kind} {placement} {_name(dtype)}", inv=inv)


UNIFORM_ROWS = ["all_nan", "all_neg_inf", "mixed_zeros"]


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("kind", UNIFORM_ROWS)
def test_rows_of_one_value(kind, dtype):
    """Every position ties (NaN of random payloads and signs, -inf, or +-0): the first n_kept positions are kept."""
    gen = torch.Generator(device=DEV).manual_seed(20 + UNIFORM_ROWS.index(kind))
    B, H, S = 2, 3, PLANT_S
    if kind == "all_nan":
        nan = torch.arange(INF_BITS[dtype] + 1, 0x8000, device=DEV)
        nan = torch.cat([nan, nan - 0x8000]).to(torch.int16)  # both signs: bits 0x8000 | m as int16
        scores = nan[torch.randint(0, nan.numel(), (B, H, S), generator=gen, device=DEV)].view(dtype)
        assert torch.isnan(scores).all()
    elif kind == "all_neg_inf":
        scores = torch.full((B, H, S), float("-inf"), dtype=dtype, device=DEV)
    else:
        scores = torch.where(torch.rand(B, H, S, generator=gen, device=DEV) < 0.5, 0.0, -0.0).to(dtype)
    k, v, kr = kv_for(B, H, S, 64, dtype, gen)
    inv = rope_inv_freq("theta1e4", 64).to(DEV)
    ns = [1, 2, TILE, TILE + 1, GROUP_TILES * TILE + 3, S // 2, S - 1, S]
    order = canonical_order(scores)
    assert torch.equal(order, torch.arange(S, device=DEV).expand(B, H, S))
    check_entry_points(scores, k, v, kr, ns, f"{kind} {_name(dtype)}", order=order, inv=inv)


# ---------------------------------------------------------------------------------------------------
# 3. shapes
# ---------------------------------------------------------------------------------------------------
SHAPES = [(S, dt) for S in SHAPE_S for dt in DTYPES]


@gpu
@pytest.mark.parametrize("S,dtype", SHAPES, ids=[f"s{S}-{_name(dt)}" for S, dt in SHAPES])
def test_sequence_lengths(S, dtype):
    gen = torch.Generator(device=DEV).manual_seed(S)
    B, H = 2, 3
    scores = mixed_scores((B, H, S), dtype, gen)
    k, v, kr = kv_for(B, H, S, 16, dtype, gen)
    inv = rope_inv_freq("theta1e4", 16).to(DEV)
    check_entry_points(scores, k, v, kr, n_kept_values(S), f"S={S} {_name(dtype)}", inv=inv)


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_flat_adakv_row(dtype):
    """The (1, 1, H·S) row AdaKV selects over, at 8 heads x 128k"""
    gen = torch.Generator(device=DEV).manual_seed(30)
    S = 8 * 131072
    scores = mixed_scores((1, 1, S), dtype, gen)
    k, v, kr = kv_for(1, 1, S, 16, dtype, gen)
    inv = rope_inv_freq("theta5e5", 16).to(DEV)
    check_entry_points(scores, k, v, kr, [1, O.kept_count(S, 0.7), S // 2, S - 1], f"flat 8x128k {_name(dtype)}", inv=inv)


@gpu
def test_select_4m_positions():
    gen = torch.Generator(device=DEV).manual_seed(31)
    S = 4 << 20
    nat = _native()
    scores = mixed_scores((1, 1, S), torch.bfloat16, gen)
    order = canonical_order(scores)
    assert torch.equal(canonical(order, S // 3).cpu(), O.select_lowest_index_ties(scores.cpu(), S // 3))
    for n in n_kept_values(S):
        assert_idx(call_select(nat, scores, n), canonical(order, n), f"select 4M n_kept={n}")


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_most_rows(dtype):
    """B·Hkv = 65535, the largest gridDim.y; 65536 is refused"""
    nat = _native()
    gen = torch.Generator(device=DEV).manual_seed(32)
    B, H, S = 3, MAX_ROWS // 3, 37
    assert B * H == MAX_ROWS
    scores = mixed_scores((B, H, S), dtype, gen)
    k, v, kr = kv_for(B, H, S, 16, dtype, gen)
    inv = rope_inv_freq("theta1e4", 16).to(DEV)
    check_entry_points(scores, k, v, kr, [1, 18, 36, 37], f"B·H={MAX_ROWS} {_name(dtype)}", inv=inv)
    with pytest.raises(RuntimeError, match="unsupported shape"):
        nat.scores_select(torch.zeros(1, MAX_ROWS + 1, 4, dtype=dtype, device=DEV), 2)


def _items(R, S):
    nt = -(-S // TILE)
    return R * (-(-nt // GROUP_TILES) + nt)


ITEM_CASES = ["two_items", "one_row_one_group", "about_one_per_sm", "about_one_wave", "many_per_cta"]


def item_shape(case: str, sm: int):
    """(B, H, S) of each work-item regime of the persistent select + compact grid"""
    if case == "two_items":
        return 1, 1, 1
    if case == "one_row_one_group":
        return 1, 1, GROUP_TILES * TILE
    if case == "about_one_per_sm":
        return 1, sm // 2, TILE
    if case == "about_one_wave":
        return 3, sm // 2, TILE - 1
    S = 8 * GROUP_TILES * TILE + 1  # 129 tiles, 9 groups: 138 items per row
    rows = -(-64 * sm // _items(1, S)) + 1
    return 2, -(-rows // 2), S


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("case", ITEM_CASES)
def test_work_item_counts(case, dtype):
    sm = _sm_count()
    B, H, S = item_shape(case, sm)
    items = _items(B * H, S)
    if case == "two_items":
        assert items == 2
    elif case == "about_one_per_sm":
        assert abs(items - sm) <= 2
    elif case == "about_one_wave":
        assert abs(items - SEL_CTAS * sm) <= 3
    elif case == "many_per_cta":
        assert items > 64 * sm
    gen = torch.Generator(device=DEV).manual_seed(33)
    scores = mixed_scores((B, H, S), dtype, gen)
    k, v, kr = kv_for(B, H, S, 16, dtype, gen)
    inv = rope_inv_freq("theta1e4", 16).to(DEV)
    check_entry_points(scores, k, v, kr, n_kept_values(S), f"{case} items={items} {_name(dtype)}", inv=inv)


@gpu
def test_n_kept_zero_launches_nothing():
    """n_kept = 0: empty outputs, and the C ABI returns before touching a null workspace or null outputs"""
    nat = _native()
    lib = nat.load()
    B, H, S, D = 2, 3, 300, 16
    gen = torch.Generator(device=DEV).manual_seed(34)
    scores = mixed_scores((B, H, S), torch.bfloat16, gen)
    k, v, kr = kv_for(B, H, S, D, torch.bfloat16, gen)
    inv = rope_inv_freq("theta1e4", D).to(DEV)
    assert call_select(nat, scores, 0).shape == (B, H, 0)
    for out in (call_compress(nat, scores, k, v, 0), call_compress(nat, scores, kr, v, 0, inv),
                call_streaming(nat, k, v, 0, 4)):
        assert [tuple(t.shape) for t in out] == [(B, H, 0, D), (B, H, 0, D), (B, H, 0)]
    p = nat.make_problem(k, v, 0)
    stride = (ctypes.c_int64 * 2)(H * S, S)
    st = nat._stream()
    assert lib.kvp_scores_select(ctypes.byref(p), scores.data_ptr(), stride, 0, 0, 0, st) == 0
    assert lib.kvp_scores_compress(ctypes.byref(p), scores.data_ptr(), stride, k.data_ptr(), v.data_ptr(),
                                   0, 0, 0, 0, 0, st) == 0
    assert lib.kvp_scores_compress_rerotate(ctypes.byref(p), scores.data_ptr(), stride, kr.data_ptr(), v.data_ptr(),
                                            inv.data_ptr(), 0, 0, 0, 0, 0, st) == 0
    assert lib.kvp_streaming_compress(ctypes.byref(p), 4, k.data_ptr(), v.data_ptr(), 0, 0, 0, st) == 0
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------
# 4. compaction: every head_dim, the copy loop's edges, K / V layouts; StreamingLLM
# ---------------------------------------------------------------------------------------------------
COMPACT_S = 3 * TILE - 5  # tiles 0 and 1 full, tile 2 padded
COMPACT_N = 300           # kept positions per row; tile 1 holds the count under test
SWEEP = [(dt, D) for dt in DTYPES for D in HEAD_DIMS]


def kv_layout(kind, B, H, S, D, dtype, gen):
    """K, V of random bit patterns laid out as `kind`; every layout is consumed in place"""
    r = lambda *s: rand_bits(s, gen, dtype)  # noqa: E731
    if kind == "contiguous":
        return r(B, H, S, D), r(B, H, S, D)
    if kind == "k_contiguous_v_bshd":
        return r(B, H, S, D), r(B, S, H, D).transpose(1, 2)
    if kind == "v_row_slice":  # rows of a wider tensor: stride D + 24, 16 bytes in
        return r(B, H, S, D), r(B, H, S, D + 24)[..., 8:8 + D]
    if kind == "k_broadcast_head":  # one head of K seen by every head (stride 0), V transposed
        return r(B, 1, S, D).expand(B, H, S, D), r(B, S, H, D).transpose(1, 2)
    n = B * H * S * D
    buf = r(2 * n + 24)  # offset_views: K 16 bytes and V 48 bytes into one buffer
    return buf[8:8 + n].view(B, H, S, D), buf[n + 24:2 * n + 24].view(B, H, S, D)


def compaction_scores(counts, dtype, gen):
    """[B, H, COMPACT_S] scores with exactly COMPACT_N positive ones per row, counts[r] of them in tile 1"""
    rows = []
    for c in counts:
        rest = COMPACT_N - c
        a = min(TILE, rest)
        hi = torch.zeros(COMPACT_S, dtype=torch.bool)
        hi[torch.randperm(TILE, generator=gen)[:a]] = True
        hi[TILE + torch.randperm(TILE, generator=gen)[:c]] = True
        hi[2 * TILE + torch.randperm(COMPACT_S - 2 * TILE, generator=gen)[:rest - a]] = True
        x = torch.rand(COMPACT_S, generator=gen) + 1
        rows.append(torch.where(hi, x, -x))
    return torch.stack(rows).to(dtype)


@gpu
@pytest.mark.parametrize("dtype,D", SWEEP, ids=[f"{_name(dt)}-d{D}" for dt, D in SWEEP])
def test_compaction(dtype, D):
    nat = _native()
    nvec = D // 8
    counts = edge_counts(nvec, SEL_U)
    B, H = 2, -(-len(counts) // 2)
    counts = (counts * 2)[:B * H]
    gen = torch.Generator().manual_seed(D)
    gen_d = torch.Generator(device=DEV).manual_seed(D)
    scores = compaction_scores(counts, dtype, gen).view(B, H, COMPACT_S).to(DEV)
    want = canonical(canonical_order(scores), COMPACT_N)
    assert torch.equal(((want >= TILE) & (want < 2 * TILE)).sum(-1).flatten().cpu(), torch.tensor(counts))
    inv = rope_inv_freq("theta1e4", D).to(DEV) if D % 16 == 0 else None
    for kind in LAYOUTS:
        k, v = kv_layout(kind, B, H, COMPACT_S, D, dtype, gen_d)
        assert nat._rows_ok(k) and nat._rows_ok(v), kind
        w = f"compaction {_name(dtype)} D={D} {kind}"
        k_out, v_out, idx = call_compress(nat, scores, k, v, COMPACT_N)
        assert_idx(idx, want, w)
        assert_gather(k_out, k, want, w + " K'")
        assert_gather(v_out, v, want, w + " V'")
        if inv is not None and kind in ("contiguous", "v_row_slice", "k_broadcast_head"):
            kr = torch.randn(B, H, COMPACT_S, D, generator=gen_d, device=DEV).to(dtype)
            k_out, v_out, idx = call_compress(nat, scores, kr, v, COMPACT_N, inv)
            assert_idx(idx, want, w + " rerotate")
            assert_gather(v_out, v, want, w + " rerotate V'")
            assert_rerotated(k_out, kr, want, inv, w)
    assert_idx(call_select(nat, scores, COMPACT_N), want, f"compaction {_name(dtype)} D={D} select")


@gpu
@pytest.mark.parametrize("dtype,D", SWEEP, ids=[f"{_name(dt)}-d{D}" for dt, D in SWEEP])
def test_streaming_compaction(dtype, D):
    """n_kept = TILE + c for every edge count c of streaming's copy loop, n_sink in {0, n_kept - 1, n_kept, > n_kept}:
    the kept ranges are the closed form, which is the canonical selection of StreamingLLM's 0 / 1 scores"""
    nat = _native()
    B, H, S = 2, 3, COMPACT_S
    gen_d = torch.Generator(device=DEV).manual_seed(100 + D)
    for kind in LAYOUTS:
        k, v = kv_layout(kind, B, H, S, D, dtype, gen_d)
        for c in edge_counts(D // 8, STREAM_U):
            n = TILE + c
            for n_sink in (0, n - 1, n, n + 7):
                scores = torch.ones(B, H, S, dtype=dtype, device=DEV)  # O.streaming_scores at this n_kept
                scores[:, :, n_sink:n_sink + S - n] = 0
                want = canonical(canonical_order(scores), n)
                assert torch.equal(want[0, 0].cpu(), O.streaming_kept(S, n, n_sink))
                w = f"streaming {_name(dtype)} D={D} {kind} n_kept={n} n_sink={n_sink}"
                k_out, v_out, idx = call_streaming(nat, k, v, n, n_sink)
                assert_idx(idx, want, w)
                assert_gather(k_out, k, want, w + " K'")
                assert_gather(v_out, v, want, w + " V'")


# ---------------------------------------------------------------------------------------------------
# 5. entry-point contracts
# ---------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_fp32_scores_are_ranked_in_the_cache_dtype(dtype):
    """fp32 scores select as scores.to(cache dtype): 1 + 2^-12 at position 900 and 1 at position 100 round to one
    tie, so n_kept = 1 keeps position 100, where an fp32 top-k would keep 900"""
    gen = torch.Generator(device=DEV).manual_seed(40)
    B, H, S = 2, 2, 3000
    x = -torch.rand(B, H, S, generator=gen, device=DEV) - 1
    x[..., 100] = 1.0
    x[..., 900] = 1.0 + 2.0 ** -12
    r = x.to(dtype)
    assert (r[..., 100] == r[..., 900]).all()
    assert not torch.equal(canonical(canonical_order(x), 1), canonical(canonical_order(r), 1))
    k, v, kr = kv_for(B, H, S, 32, dtype, gen)
    inv = rope_inv_freq("theta1e4", 32).to(DEV)
    nat = _native()
    order = canonical_order(r)
    for n in (1, 2, 1500, S):
        want = canonical(order, n)
        k_out, v_out, idx = call_compress(nat, x, k, v, n)
        assert_idx(idx, want, f"fp32 scores n_kept={n}")
        assert_gather(k_out, k, want, "fp32 scores K'")
        assert_gather(v_out, v, want, "fp32 scores V'")
        k_out, v_out, idx = call_compress(nat, x, kr, v, n, inv)
        assert_idx(idx, want, f"fp32 scores rerotate n_kept={n}")
        assert_rerotated(k_out, kr, want, inv, "fp32 scores rerotate")
    assert int(call_compress(nat, x, k, v, 1)[2][0, 0, 0]) == 100


SCORE_STRIDES = ["every_other_head", "broadcast_over_b", "broadcast_over_h", "transposed"]


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("kind", SCORE_STRIDES)
def test_score_strides(kind, dtype):
    gen = torch.Generator(device=DEV).manual_seed(41 + SCORE_STRIDES.index(kind))
    B, H, S = 3, 4, 2 * GROUP_TILES * TILE + 3
    if kind == "every_other_head":
        scores = mixed_scores((B, 2 * H, S), dtype, gen)[:, ::2]
    elif kind == "broadcast_over_b":
        scores = mixed_scores((1, H, S), dtype, gen).expand(B, H, S)
    elif kind == "broadcast_over_h":
        scores = mixed_scores((B, 1, S), dtype, gen).expand(B, H, S)
    else:
        scores = mixed_scores((B, S, H), dtype, gen).transpose(1, 2)
    assert not scores.is_contiguous()
    k, v, kr = kv_for(B, H, S, 32, dtype, gen)
    inv = rope_inv_freq("theta1e4", 32).to(DEV)
    check_entry_points(scores, k, v, kr, n_kept_values(S), f"score strides {kind} {_name(dtype)}", inv=inv)


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_graph_replay_with_scores_updated_in_place(dtype):
    nat = _native()
    gen = torch.Generator(device=DEV).manual_seed(50)
    B, H, S, D, n = 2, 3, 9000, 32, 4000
    scores = mixed_scores((B, H, S), dtype, gen)
    k, v, kr = kv_for(B, H, S, D, dtype, gen)
    inv = rope_inv_freq("theta1e4", D).to(DEV)
    graphed = nat.capture(lambda: (nat.scores_select(scores, n),
                                   *nat.scores_compress(scores, k, v, n, return_indices=True),
                                   *nat.scores_compress_rerotate(scores, kr, v, n, inv, return_indices=True)))
    for seed in (51, 52):
        scores.copy_(mixed_scores((B, H, S), dtype, torch.Generator(device=DEV).manual_seed(seed)))
        sel, k_out, v_out, idx, kr_out, vr_out, idx_r = graphed.replay()
        torch.cuda.synchronize()
        want = canonical(canonical_order(scores), n)
        for i, w in ((sel, "select"), (idx, "compress"), (idx_r, "rerotate")):
            assert_idx(i, want, f"graph replay {w} seed {seed}")
        assert_gather(k_out, k, want, "graph replay K'")
        assert_gather(v_out, v, want, "graph replay V'")
        assert_gather(vr_out, v, want, "graph replay rerotate V'")
        assert_rerotated(kr_out, kr, want, inv, "graph replay rerotate")
        eager = call_compress(nat, scores, k, v, n)
        assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(eager[:2], (k_out, v_out)))


@gpu
def test_growing_and_shrinking_shapes_on_one_stream():
    """Calls of growing, shrinking, then growing shapes enqueued back to back: the cached workspace grows, and each
    call's memset clears its own zeroed region of the reused buffer, whatever an earlier, larger call left there"""
    nat = _native()
    gen = torch.Generator(device=DEV).manual_seed(60)
    shapes = [(2, 3, 5000), (4, 8, 40000), (1, 2, 300), (2, 2, 1), (8, 8, 70000), (3, 5, 20000)]
    inputs = []
    for B, H, S in shapes:
        scores = mixed_scores((B, H, S), torch.float16, gen)
        inputs.append((scores, *kv_for(B, H, S, 16, torch.float16, gen)[:2], max(1, S // 3)))
    torch.cuda.synchronize()
    calls = []
    for scores, k, v, n in inputs:  # no synchronisation in between
        out = call_compress(nat, scores, k, v, n, check=False)
        calls.append((scores, k, v, n, out, call_select(nat, scores, n, check=False)))
    _check_ws(nat, _select_problem(nat, inputs[-1][0], inputs[-1][3]))  # the last call; it synchronises
    for scores, k, v, n, (k_out, v_out, idx), sel in calls:
        want = canonical(canonical_order(scores), n)
        what = f"back to back {tuple(scores.shape)}"
        assert_idx(idx, want, what)
        assert_idx(sel, want, what + " select")
        assert_gather(k_out, k, want, what + " K'")
        assert_gather(v_out, v, want, what + " V'")


@gpu
def test_two_streams_concurrently():
    """Large calls on two streams at once, each with its own cached workspace, equal the same calls run serially"""
    nat = _native()
    gen = torch.Generator(device=DEV).manual_seed(70)
    B, H, S, D = 2, 8, 100000, 16
    n = S // 2
    inputs = []
    for _ in range(2):
        scores = mixed_scores((B, H, S), torch.bfloat16, gen)
        inputs.append((scores, *kv_for(B, H, S, D, torch.bfloat16, gen)[:2]))
    serial = [call_compress(nat, sc, k, v, n) for sc, k, v in inputs]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for s in streams:
        s.wait_stream(torch.cuda.current_stream())
    outs = []
    for _ in range(3):  # repeated, so the streams' calls overlap
        for s, (sc, k, v) in zip(streams, inputs):
            with torch.cuda.stream(s):
                outs.append(call_compress(nat, sc, k, v, n, check=False))
    torch.cuda.synchronize()
    workspaces = set()
    for s, (sc, k, v) in zip(streams, inputs):
        with torch.cuda.stream(s):
            p = nat.make_problem(k, v, n)
            _check_ws(nat, p)
            workspaces.add(nat._workspace(p, nat.SCORER_GENERIC, torch.device(DEV)).data_ptr())
    assert len(workspaces) == 2, "the two streams share a workspace"
    for i, out in enumerate(outs):
        ref = serial[i % 2]
        assert torch.equal(out[2], ref[2]) and all(torch.equal(_bits(a), _bits(b)) for a, b in zip(out[:2], ref[:2])), \
            f"stream call {i} differs from the serial call"
    for (sc, k, v), (k_out, v_out, idx) in zip(inputs, serial):
        want = canonical(canonical_order(sc), n)
        assert_idx(idx, want, "serial call")
        assert_gather(k_out, k, want, "serial call K'")
        assert_gather(v_out, v, want, "serial call V'")
