"""FinchPress's chunked selection and compaction against an exact reference: every 16-bit key, every chunk edge, every
head_dim, through the caller-scores entry point `kvp_scores_compress_chunked`.

Two kernels of select_compact.cu do the work. `chunk_select_kernel` (one CTA per (chunk, row)) finds each chunk's exact
16-bit threshold from two 256-bin histograms, then writes the kept positions in position order, walking the chunk in
256-position tiles that carry `kept_before` / `eq_before` from tile to tile. `chunk_gather_kernel` (one CTA per 256
output rows of a row: a gather item) copies the kept K / V rows, or re-rotates the keys by the global delta j - s
starting at its first output row j0. The contract is the selection sweep's (tests/test_gpu_select_compact_sweep.py),
applied per chunk: chunk c holds positions [c L, min(S, (c + 1) L)); each of the S // L full chunks keeps its
chunk_kept largest scores in the cache dtype, the short last chunk (S % L positions) its tail_kept, ties to the lowest
position, -0 == +0, NaN of either sign above +inf; chunk c's kept positions, ascending, go to output rows
[c chunk_kept, (c + 1) chunk_kept). So every bar is exact:
  * `idx` is int32 and equals the chunked canonical selection (`gpu_support.chunked_canonical`: per chunk the stable
    descending sort of the oracle's key, the first chunk_kept / tail_kept, ascending, plus the chunk's start); each test
    checks one case against `oracle.press_oracle.select_lowest_index_ties` applied chunk by chunk;
  * K' and V' are bitwise gathers (K and V hold random bit patterns, NaN payloads included);
  * a re-rotated K' is one of the admissible roundings of `gpu_support.rerotation_admissible` at the global output
    position j;
  * outputs are poisoned before each call (0xFF blocks, `gpu_support._poison`), and `native.workspace_check` runs after
    the calls.
The edge cases call the C ABI with explicit chunk_length / chunk_kept / tail_kept (`call_chunked`); the Python wrapper
only derives them from a compression ratio.

The cases: (1) a chunk holding all 65536 patterns of a dtype, chunk_kept at every high-byte bin boundary and +-1 and at
every low-byte boundary of the NaN, +-inf, zero and subnormal bins, and rows of several such chunks, each its own
permutation, with a short tail chunk; (2) planted threshold ties (negative, mixed-sign, NaN, low bytes 0x00 / 0xFF)
straddling the 256-position tiles inside every chunk or only in the tail chunk, and chunks of all NaN, all -inf or mixed
+-0; (3) chunk lengths 1, 2, 255-257, 511-513, S - 1, S, S + 1 with tails 0, 1 and L - 1, chunk_kept in {1, L}, tail_kept
in {1, tail}, no full chunk (L > S) with a chunk_kept the kernels must ignore, kept counts on both sides of 256, 512 and
768 (gather items and their j0), L = 1 at S = 131072 (gridDim.x = 131072) and B·Hkv = 65535; (4) a single chunk is
bitwise `scores_compress` / `scores_compress_rerotate`, chunks kept whole give idx = arange(S) and K' = K (re-rotated by
delta 0 too), and a null idx_out changes no K' / V' bit; (5) every head_dim 8..256 with each gather item's kept count at
the batch edges of copy_rows_kv<kSelU>, through the five K / V layouts of `gpu_support.LAYOUTS`, and re-rotation at every
D % 16 == 0 in both dtypes; (6) fp32 and strided scores, an exact-size 0xFF-filled workspace and the smallest one the
entry point accepts, graph replay with the scores updated in place, two streams. CPU tests check that the tile,
gather-item and copy-edge constants the case lists use are the sources', and the reference shortcut against the oracle.

On an H100 80GB HBM3 (700 W power limit) the 157 GPU cases here and the 114 of tests/test_gpu_finch_fallback_sweep.py
pass in about 80 s together. No case found a kernel bug. Ranking -0 below +0 in the keys, or starting the gather's
re-rotation at output row 0 instead of j0, fails test_key_space_one_chunk.
"""
import re
from pathlib import Path

import pytest
import torch

from kvpress_b200 import native
from tests.gpu_support import (INF_BITS, LAYOUTS, TILE, TILE_THREADS, _bits, _kv_out_bytes, _landed, _layout, _name,
                               _native, _pattern_keys, _poison, _score_copy_bytes, all_patterns, assert_gather,
                               assert_idx, chunk_orders, chunked_canonical, chunked_from_orders,
                               chunked_oracle, copy_edges, edge_counts, key16, key_space_n_kept, kv_for, mixed_scores,
                               rand_bits, rerotation_admissible, rope_inv_freq, threshold_patterns)

gpu = pytest.mark.gpu
DEV = "cuda:0"
CSRC = Path(__file__).resolve().parent.parent / "kvpress_b200" / "csrc"
DTYPES = [torch.bfloat16, torch.float16]

# the constants of common.cuh / select_compact.cu the case lists are derived from (checked by a CPU test)
SEL_U = 3          # kSelU: copy_rows_kv<kSelU> of chunk_gather_kernel
ITEM_ROWS = TILE   # output rows per gather item (kTile); chunk_select_kernel walks a chunk in TILE_THREADS positions
MAX_ROWS = 65535   # B·Hkv: gridDim.y


# ---------------------------------------------------------------------------------------------------
# calls: explicit chunk counts, poisoned outputs, workspace check
# ---------------------------------------------------------------------------------------------------
def n_kept_of(S, L, ck, tk):
    return (S // L) * ck + tk if S >= L else tk


def _chunked(scores, k, v, L, ck, tk, inv=None, with_idx=True):
    """kvp_scores_compress_chunked with these chunk counts, as native.scores_compress_chunked makes the call"""
    nat = _native()
    sc, sstride = nat._caller_scores(scores, k)
    return nat._compress("kvp_scores_compress_chunked", nat.SCORER_FINCH, k, v, n_kept_of(k.shape[2], L, ck, tk),
                         (sc, sstride, L, ck, tk, k, v, nat._inv_freq(inv, k)), with_idx)


def _check_ws(k, v, n):
    nat = _native()
    p = nat.make_problem(k, v, n)
    nat.workspace_check(p, nat.SCORER_FINCH, nat._workspace(p, nat.SCORER_FINCH, torch.device(DEV)))


def call_chunked(scores, k, v, L, ck, tk, inv=None, with_idx=True, check=False):
    """One poisoned call; `check`: workspace_check after it (it synchronises the stream)"""
    assert native._rows_ok(k) and native._rows_ok(v), "K / V would be copied, not consumed in place"
    n = n_kept_of(k.shape[2], L, ck, tk)
    ptrs = _poison(_score_copy_bytes(scores, k.dtype), *_kv_out_bytes(k, n)[: 3 if with_idx else 2])
    out = _chunked(scores, k, v, L, ck, tk, inv, with_idx)
    _landed(ptrs, *out)
    if check:
        _check_ws(k, v, n)
    return out


def assert_rerotated(k_out, k, want, inv, what):
    adm = _bits(rerotation_admissible(k, want, inv))
    hit = (adm == _bits(k_out)[None]).any(0)
    assert hit.all(), f"{what}: {int((~hit).sum())} of {hit.numel()} re-rotated K' elements not admissible"


def check_counts(scores, k, v, L, counts, what, orders=None, kr=None, inv=None, rerotate_every=1):
    """Every (chunk_kept, tail_kept) of `counts` through the plain call (K / V) and, on every `rerotate_every`-th, the
    re-rotating call (kr / V); one case against the oracle chunk by chunk; workspace_check after the last call."""
    orders = chunk_orders(scores, L) if orders is None else orders
    ck0, tk0 = counts[len(counts) // 2]
    S = k.shape[2]
    # the oracle on the scores in the cache dtype, one call per chunk: on the first 256 chunks of a row of more
    m = S if S // L <= 256 else 256 * L
    ref = chunked_oracle(scores[..., :m].to(k.dtype), L, ck0, tk0 if m == S else 0)
    assert torch.equal(chunked_from_orders(orders, L, ck0, tk0)[..., : ref.shape[-1]].cpu(), ref), what
    for i, (ck, tk) in enumerate(counts):
        w = f"{what} L={L} chunk_kept={ck} tail_kept={tk}"
        want = chunked_from_orders(orders, L, ck, tk)
        k_out, v_out, idx = call_chunked(scores, k, v, L, ck, tk)
        assert_idx(idx, want, w)
        assert_gather(k_out, k, want, w + " K'")
        assert_gather(v_out, v, want, w + " V'")
        if inv is not None and i % rerotate_every == 0:
            k_out, v_out, idx = call_chunked(scores, kr, v, L, ck, tk, inv)
            assert_idx(idx, want, w + " rerotate")
            assert_gather(v_out, v, want, w + " rerotate V'")
            assert_rerotated(k_out, kr, want, inv, w + " rerotate")
    _check_ws(k, v, n_kept_of(k.shape[2], L, *counts[-1]))


def bits_of(x, gen):
    """K or V in one of gpu_support.LAYOUTS, overwritten in place with random bit patterns (NaN payloads included)"""
    x.view(torch.int16).copy_(rand_bits(x.shape, gen, x.dtype).view(torch.int16))
    return x


# ---------------------------------------------------------------------------------------------------
# CPU: the case lists follow the sources' constants; the reference shortcut is the oracle
# ---------------------------------------------------------------------------------------------------
def _constant(text: str, name: str) -> int:
    m = re.search(rf"constexpr\s+\w+\s+{name}\s*=\s*(\w+)", text)
    assert m, name
    return int(m.group(1), 0)


def _kernel(text: str, name: str) -> str:
    return re.search(rf"{name}\(.*?\n}}", text, re.S).group(0)


def test_case_lists_follow_the_source_constants():
    common = (CSRC / "common.cuh").read_text()
    sc = (CSRC / "select_compact.cu").read_text()
    assert _constant(common, "kTile") == TILE == ITEM_ROWS and _constant(common, "kTileThreads") == TILE_THREADS
    assert _constant(sc, "kSelU") == SEL_U
    select = _kernel(sc, "chunk_select_kernel")
    # the three passes over a chunk step by one tile of TILE_THREADS positions, carrying the counts across tiles
    assert select.count("base += kTileThreads") == 3 and "kept_before +=" in select and "eq_before +=" in select
    assert "c < S / L ? (uint32_t)chunk_kept : (uint32_t)tail_kept" in select
    gather = _kernel(sc, "chunk_gather_kernel")
    assert "j0 = blockIdx.x * kTile" in gather and "min(kTile, n_kept - j0)" in gather
    assert "copy_rows_kv<kSelU>(" in gather and re.search(r"copy_rows_k_rerotated<TR>\([^;]*\bj0\);", gather, re.S)
    launch = _kernel(sc, "launch_select_compact_chunked")
    assert "(d.n_kept + kTile - 1) / kTile" in launch and "dim3(n_chunks, d.R)" in launch
    assert "p->B * p->Hkv > 65535" in (CSRC / "api.cu").read_text()
    # chunk lengths on both sides of one and two tiles; kept counts on both sides of one, two and three gather items
    assert {TILE - 1, TILE, TILE + 1, 2 * TILE - 1, 2 * TILE, 2 * TILE + 1} <= set(L for L, _ in GEOMETRY)
    for e in (ITEM_ROWS, 2 * ITEM_ROWS, 3 * ITEM_ROWS):
        assert {e - 1, e, e + 1} <= set(ITEM_N)
    # per head_dim, the kept counts of the last gather item straddle every copy edge of copy_rows_kv<kSelU>
    for nvec in range(1, 33):
        cs = edge_counts(nvec, SEL_U)
        for e in copy_edges(SEL_U):
            at = -(-e // nvec)
            if at + 1 <= ITEM_ROWS:
                assert {(e - 1) // nvec, at, e // nvec + 1} <= set(cs)
        for c in cs:  # compaction_counts places them in the second item
            ck, tk = compaction_counts(ITEM_ROWS + c)
            assert 1 <= ck <= COMPACT_L and 1 <= tk <= COMPACT_S % COMPACT_L
            assert 3 * ck + tk == ITEM_ROWS + c


def test_chunked_reference_is_the_oracle():
    """chunked_canonical == select_lowest_index_ties applied chunk by chunk, on rows full of ties and special values"""
    g = torch.Generator().manual_seed(3)
    for dtype in DTYPES:
        row = all_patterns(dtype)[torch.randint(0, 65536, (2, 3, 700), generator=g)]
        row[..., ::3] = torch.tensor([0.0, -0.0, float("nan"), float("-inf")], dtype=dtype)[
            torch.randint(0, 4, (2, 3, 234), generator=g)]
        for L in (1, 7, 256, 699, 700, 701, 5000):
            n_full, tail = divmod(700, L)
            for ck in {1, L // 2 or 1, L} if n_full else {-3}:
                for tk in {1, tail // 2 or 1, tail} if tail else {0}:
                    assert torch.equal(chunked_canonical(row, L, ck, tk), chunked_oracle(row, L, ck, tk)), (L, ck, tk)


# ---------------------------------------------------------------------------------------------------
# 1. the whole key space
# ---------------------------------------------------------------------------------------------------
def _permuted_patterns(dtype, n_chunks, rows, gen):
    pats = all_patterns(dtype).to(DEV)
    return torch.stack([torch.cat([pats[torch.randperm(65536, generator=gen, device=DEV)] for _ in range(n_chunks)])
                        for _ in range(rows)])


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_name)
def test_key_space_one_chunk(dtype):
    """Two rows whose first chunk holds all 65536 patterns (a permutation each) and whose tail chunk holds 300 random
    ones; chunk_kept at every boundary of key_space_n_kept."""
    gen = torch.Generator(device=DEV).manual_seed(100)
    L, tail = 65536, 300
    scores = torch.cat([_permuted_patterns(dtype, 1, 2, gen), rand_bits((2, tail), gen, dtype)], -1).view(1, 2, -1)
    S = scores.shape[-1]
    k, v, kr = kv_for(1, 2, S, 16, dtype, gen)
    inv = rope_inv_freq("theta1e4", 16).to(DEV)
    cks = key_space_n_kept(key16(all_patterns(dtype).view(torch.int16), dtype), dtype)
    tks = (1, tail // 2, tail)
    counts = [(ck, tks[i % 3]) for i, ck in enumerate(cks)]
    check_counts(scores, k, v, L, counts, f"key space {_name(dtype)}", kr=kr, inv=inv, rerotate_every=8)


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_name)
def test_key_space_several_chunks(dtype):
    """Rows of three chunks, each its own permutation of all 65536 patterns, and a tail chunk of 1000"""
    gen = torch.Generator(device=DEV).manual_seed(101)
    L, tail = 65536, 1000
    scores = torch.cat([_permuted_patterns(dtype, 3, 2, gen), rand_bits((2, tail), gen, dtype)], -1).view(2, 1, -1)
    S = scores.shape[-1]
    k, v, kr = kv_for(2, 1, S, 16, dtype, gen)
    inv = rope_inv_freq("theta5e5", 16).to(DEV)
    cks = key_space_n_kept(key16(all_patterns(dtype).view(torch.int16), dtype), dtype)[::7]
    tks = (1, 499, tail)
    counts = [(ck, tks[i % 3]) for i, ck in enumerate(cks)]
    check_counts(scores, k, v, L, counts, f"key space x3 {_name(dtype)}", kr=kr, inv=inv, rerotate_every=10)


# ---------------------------------------------------------------------------------------------------
# 2. planted threshold ties
# ---------------------------------------------------------------------------------------------------
PL, P_TAIL = 1000, 300     # chunk length and tail of the planted rows: chunks of four tiles, the last one partial
PS = 3 * PL + P_TAIL
THRESHOLDS = ["neg_inf", "most_negative", "nan", "key_lo00", "key_loff", "zero_mixed_sign"]
PLACEMENTS = ["straddle_tiles", "tail_only"]
PLANTED = [(t, p, dt) for t in THRESHOLDS for p in PLACEMENTS for dt in DTYPES]


def planted_chunk(kind, length, tie_pos, dtype, gen):
    """One chunk: the threshold key at tie_pos, every other position strictly above or below it. Returns (int16
    patterns, n_gt)."""
    pats, keys = _pattern_keys(dtype)
    tie_pats = threshold_patterns(kind, dtype)
    T = int(key16(tie_pats[:1], dtype))
    above, below = pats[keys > T], pats[keys < T]
    rest = torch.ones(length, dtype=torch.bool)
    rest[tie_pos] = False
    rest = rest.nonzero()[:, 0]
    rest = rest[torch.randperm(rest.numel(), generator=gen)]
    n_gt = 0 if above.numel() == 0 else rest.numel() if below.numel() == 0 else rest.numel() // 2
    row = torch.empty(length, dtype=torch.int16)
    row[tie_pos] = tie_pats[torch.randint(0, tie_pats.numel(), (len(tie_pos),), generator=gen)]
    if n_gt:
        row[rest[:n_gt]] = above[torch.randint(0, above.numel(), (n_gt,), generator=gen)]
    n_lt = rest.numel() - n_gt
    if n_lt:
        row[rest[n_gt:]] = below[torch.randint(0, below.numel(), (n_lt,), generator=gen)]
    return row, n_gt


def _straddle(centres, half):
    return torch.cat([torch.arange(c - half, c + half) for c in centres])


@gpu
@pytest.mark.parametrize("kind,placement,dtype", PLANTED, ids=[f"{k}-{p}-{_name(dt)}" for k, p, dt in PLANTED])
def test_planted_threshold_ties(kind, placement, dtype):
    """The tail chunk's ties straddle its first tile edge; with "straddle_tiles" every full chunk's ties straddle its
    first and second tile edges, with "tail_only" the full chunks hold random patterns. chunk_kept / tail_kept take one
    tie, half, all but one and all of them."""
    gen = torch.Generator().manual_seed(200 + 10 * THRESHOLDS.index(kind) + PLACEMENTS.index(placement))
    rows, n_gt_full, n_gt_tail = [], set(), set()
    full_ties, tail_ties = _straddle((TILE, 2 * TILE), 10), _straddle((TILE,), 10)
    for _ in range(4):
        parts = []
        for _c in range(3):
            if placement == "straddle_tiles":
                part, n_gt = planted_chunk(kind, PL, full_ties, dtype, gen)
                n_gt_full.add(n_gt)
            else:
                part = torch.randint(-32768, 32768, (PL,), generator=gen, dtype=torch.int16)
            parts.append(part)
        part, n_gt = planted_chunk(kind, P_TAIL, tail_ties, dtype, gen)
        n_gt_tail.add(n_gt)
        rows.append(torch.cat(parts + [part]))
    assert len(n_gt_tail) == 1 and len(n_gt_full) <= 1
    scores = torch.stack(rows).view(dtype).view(2, 2, PS).to(DEV)
    nt, nf = tail_ties.numel(), full_ties.numel()
    tks = [next(iter(n_gt_tail)) + t for t in (1, nt // 2, nt - 1, nt)]
    if n_gt_full:
        g = next(iter(n_gt_full))
        cks = [g + t for t in (1, nf // 2, nf - 1, nf)]
    else:
        cks = [1, PL // 2, PL - 1, PL]
    if kind in ("nan", "zero_mixed_sign"):  # both signs among the ties
        tie = scores[..., 3 * PL:].view(torch.int16)[..., tail_ties]
        assert (tie < 0).any() and (tie >= 0).any()
    gen_d = torch.Generator(device=DEV).manual_seed(11)
    k, v, kr = kv_for(2, 2, PS, 64, dtype, gen_d)
    inv = rope_inv_freq("theta5e5", 64).to(DEV)
    check_counts(scores, k, v, PL, list(zip(cks, tks)), f"planted {kind} {placement} {_name(dtype)}", kr=kr, inv=inv)


UNIFORM = ["all_nan", "all_neg_inf", "mixed_zeros"]


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_name)
@pytest.mark.parametrize("kind", UNIFORM)
def test_chunks_of_one_value(kind, dtype):
    """Every position ties (NaN of random payloads and signs, -inf, or +-0): each chunk keeps its first positions"""
    gen = torch.Generator(device=DEV).manual_seed(300 + UNIFORM.index(kind))
    B, H = 2, 3
    if kind == "all_nan":
        nan = torch.arange(INF_BITS[dtype] + 1, 0x8000, device=DEV)
        nan = torch.cat([nan, nan - 0x8000]).to(torch.int16)
        scores = nan[torch.randint(0, nan.numel(), (B, H, PS), generator=gen, device=DEV)].view(dtype)
        assert torch.isnan(scores).all()
    elif kind == "all_neg_inf":
        scores = torch.full((B, H, PS), float("-inf"), dtype=dtype, device=DEV)
    else:
        scores = torch.where(torch.rand(B, H, PS, generator=gen, device=DEV) < 0.5, 0.0, -0.0).to(dtype)
    orders = chunk_orders(scores, PL)
    assert torch.equal(orders[0], torch.arange(PL, device=DEV).expand(B, H, 3, PL))
    k, v, kr = kv_for(B, H, PS, 64, dtype, gen)
    inv = rope_inv_freq("theta1e4", 64).to(DEV)
    counts = [(1, 1), (TILE - 1, TILE), (TILE, TILE + 1), (TILE + 1, P_TAIL - 1), (PL - 1, 2), (PL, P_TAIL)]
    check_counts(scores, k, v, PL, counts, f"{kind} {_name(dtype)}", orders=orders, kr=kr, inv=inv)


# ---------------------------------------------------------------------------------------------------
# 3. chunk geometry
# ---------------------------------------------------------------------------------------------------
GEOM_S = 1500


def _geometry():
    """(L, S): each chunk length with S of tail 0, 1 and L - 1, and chunk lengths past S (no full chunk)"""
    out = []
    for L in (1, 2, TILE - 1, TILE, TILE + 1, 2 * TILE - 1, 2 * TILE, 2 * TILE + 1, GEOM_S - 1, GEOM_S, GEOM_S + 1):
        m = max(1, GEOM_S // L)
        out += sorted({(L, S) for S in (m * L, m * L + 1, m * L + L - 1)} - set(out))
    return out + [(GEOM_S + 1, GEOM_S), (2 ** 31 - 1, 777), (2 * TILE + 1, 2 * TILE)]


GEOMETRY = _geometry()
ITEM_N = [TILE - 1, TILE, TILE + 1, 2 * TILE - 1, 2 * TILE, 2 * TILE + 1, 3 * TILE - 1, 3 * TILE, 3 * TILE + 1]


def geometry_counts(S, L):
    """chunk_kept in {1, L, half}, tail_kept in {1, tail, half}; with no full chunk, chunk_kept values the kernels
    must ignore"""
    n_full, tail = divmod(S, L)
    cks = sorted({1, L, (L + 1) // 2}) if n_full else [-3, 0, 2 ** 30]
    tks = sorted({1, tail, (tail + 1) // 2}) if tail else [0]
    return [(ck, tk) for ck in cks for tk in tks]


@gpu
@pytest.mark.parametrize("L,S", GEOMETRY, ids=[f"L{L}-S{S}" for L, S in GEOMETRY])
def test_chunk_geometry(L, S):
    dtype = DTYPES[GEOMETRY.index((L, S)) % 2]
    gen = torch.Generator(device=DEV).manual_seed(400 + GEOMETRY.index((L, S)))
    scores = mixed_scores((1, 3, S), dtype, gen)
    k, v, kr = kv_for(1, 3, S, 16, dtype, gen)
    inv = rope_inv_freq("theta1e4", 16).to(DEV)
    check_counts(scores, k, v, L, geometry_counts(S, L), f"geometry {_name(dtype)} S={S}", kr=kr, inv=inv)


COMPACT_L = 200                     # chunk length of the gather-item cases: three full chunks and a tail of 199
COMPACT_S = 4 * COMPACT_L - 1


def compaction_counts(n):
    """(chunk_kept, tail_kept) of COMPACT_S positions in chunks of COMPACT_L that keep n in all"""
    ck = min(COMPACT_L, (n - 1) // 3)
    return ck, n - 3 * ck


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_name)
def test_gather_items(dtype):
    """n_kept on both sides of one, two and three gather items of 256 output rows: each item's j0 is crossed"""
    gen = torch.Generator(device=DEV).manual_seed(500)
    scores = mixed_scores((2, 2, COMPACT_S), dtype, gen)
    k, v, kr = kv_for(2, 2, COMPACT_S, 32, dtype, gen)
    inv = rope_inv_freq("random_first_one", 32, seed=5).to(DEV)
    check_counts(scores, k, v, COMPACT_L, [compaction_counts(n) for n in ITEM_N], f"items {_name(dtype)}", kr=kr,
                 inv=inv)


@gpu
def test_one_position_chunks_at_128k():
    """L = 1 at S = 131072: gridDim.x = 131072 chunks, every position kept, 512 gather items per row"""
    gen = torch.Generator(device=DEV).manual_seed(501)
    S = 131072
    scores = mixed_scores((1, 2, S), torch.bfloat16, gen)
    k, v, kr = kv_for(1, 2, S, 16, torch.bfloat16, gen)
    inv = rope_inv_freq("theta5e5", 16).to(DEV)
    check_counts(scores, k, v, 1, [(1, 0)], "L=1 S=128k", kr=kr, inv=inv)


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_name)
def test_most_rows(dtype):
    """B·Hkv = 65535, the largest gridDim.y of both kernels"""
    gen = torch.Generator(device=DEV).manual_seed(502)
    B, H, S, L = 3, MAX_ROWS // 3, 37, 10
    assert B * H == MAX_ROWS
    scores = mixed_scores((B, H, S), dtype, gen)
    k, v, kr = kv_for(B, H, S, 16, dtype, gen)
    inv = rope_inv_freq("theta1e4", 16).to(DEV)
    check_counts(scores, k, v, L, [(1, 1), (4, 3), (L, 7)], f"B·H={MAX_ROWS} {_name(dtype)}", kr=kr, inv=inv)


# ---------------------------------------------------------------------------------------------------
# 4. equivalences
# ---------------------------------------------------------------------------------------------------
def _same_outputs(a, b, what):
    for x, y, name in zip(a, b, ("K'", "V'", "idx")):
        if x is None or y is None:
            continue
        assert torch.equal(_bits(x) if x.dtype != torch.int32 else x, _bits(y) if y.dtype != torch.int32 else y), \
            f"{what}: {name} differs"


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_name)
def test_one_chunk_is_the_unchunked_selection(dtype):
    """L = S with chunk_kept = n, and L > S with tail_kept = n, are bitwise scores_compress / _rerotate"""
    nat = _native()
    gen = torch.Generator(device=DEV).manual_seed(600)
    B, H, S = 2, 2, 3000
    scores = mixed_scores((B, H, S), dtype, gen)
    k, v, kr = kv_for(B, H, S, 64, dtype, gen)
    inv = rope_inv_freq("theta1e4", 64).to(DEV)
    for n in (1, 700, S - 1, S):
        plain = nat.scores_compress(scores, k, v, n, return_indices=True)
        rerot = nat.scores_compress_rerotate(scores, kr, v, n, inv, return_indices=True)
        for L, ck, tk in ((S, n, 0), (S + 5, 7, n)):
            w = f"{_name(dtype)} n={n} L={L}"
            _same_outputs(call_chunked(scores, k, v, L, ck, tk), plain, w)
            _same_outputs(call_chunked(scores, kr, v, L, ck, tk, inv), rerot, w + " rerotate")
    assert_idx(plain[2], chunked_canonical(scores, S, S, 0), "n=S")
    _check_ws(k, v, S)


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_name)
def test_chunks_kept_whole(dtype):
    """chunk_kept = L and tail_kept = tail keep every position: idx = arange(S), K' = K and V' = V bitwise, and the
    re-rotated K' = K too (delta 0: cos 1, sin 0; the keys are finite and nonzero)"""
    gen = torch.Generator(device=DEV).manual_seed(601)
    B, H, S = 1, 3, 1500
    scores = mixed_scores((B, H, S), dtype, gen)
    k, v, kr = kv_for(B, H, S, 128, dtype, gen)
    assert (kr != 0).all()
    inv = rope_inv_freq("yarn_like", 128).to(DEV)
    for L in (1, TILE, 700, S, S + 1):
        n_full, tail = divmod(S, L)
        ck = L if n_full else 5
        k_out, v_out, idx = call_chunked(scores, k, v, L, ck, tail)
        assert torch.equal(idx.long(), torch.arange(S, device=DEV).expand(B, H, S)), f"L={L}"
        assert torch.equal(_bits(k_out), _bits(k)) and torch.equal(_bits(v_out), _bits(v)), f"L={L}"
        kr_out, vr_out, _ = call_chunked(scores, kr, v, L, ck, tail, inv)
        assert torch.equal(_bits(kr_out), _bits(kr)) and torch.equal(_bits(vr_out), _bits(v)), f"L={L} rerotate"
    _check_ws(k, v, S)


@gpu
@pytest.mark.parametrize("rerotate", [False, True], ids=["copy", "rerotate"])
def test_null_idx_out_changes_nothing(rerotate):
    """Finch compress and the caller-scores entry point with idx_out null give the K' and V' they give with it set"""
    g = torch.Generator(device=DEV).manual_seed(602)
    B, H, G, S, D, w = 1, 2, 4, 3001, 128, 40
    k = torch.randn(B, H, S, D, generator=g, device=DEV).to(torch.float16)
    v = torch.randn(B, H, S, D, generator=g, device=DEV).to(torch.float16)
    q = (torch.randn(B, H * G, w, D, generator=g, device=DEV) * 1.5).to(torch.float16)
    inv = rope_inv_freq("theta10000", D).to(DEV) if rerotate else None
    for L in (None, 300, 1024):
        with_idx = native.finch_compress(k, v, q, w, 0.5, L, True, inv, True, True)
        without = native.finch_compress(k, v, q, w, 0.5, L, True, inv, False, True)
        assert without[2] is None
        _same_outputs(without[:2], with_idx[:2], f"finch L={L}")
        _, ck, tk, n = native.chunk_counts(S, L, 0.5)
        scores = with_idx[3].clone()
        scores[..., -w:] = float("inf")  # the window is forced
        assert_idx(with_idx[2], chunked_canonical(scores, L, ck, tk) if L else chunked_canonical(scores, S, n, 0),
                   f"finch L={L}")
    scores = mixed_scores((B, H, S), torch.float16, g)
    for L, ck, tk in ((300, 150, 1), (1024, 1, 953)):
        a = call_chunked(scores, k, v, L, ck, tk, inv)
        b = call_chunked(scores, k, v, L, ck, tk, inv, with_idx=False)
        _same_outputs(b[:2], a[:2], f"chunked L={L}")
    _check_ws(k, v, n_kept_of(S, 1024, 1, 953))


# ---------------------------------------------------------------------------------------------------
# 5. compaction: every head_dim, each gather item's copy edges, K / V layouts
# ---------------------------------------------------------------------------------------------------
HEAD_DIMS = list(range(8, 257, 8))
SWEEP = [(dt, D) for dt in DTYPES for D in HEAD_DIMS]


@gpu
@pytest.mark.parametrize("dtype,D", SWEEP, ids=[f"{_name(dt)}-d{D}" for dt, D in SWEEP])
def test_compaction(dtype, D):
    """n_kept = 256 + c: the second gather item copies c rows, for every c at the batch edges of copy_rows_kv<kSelU>;
    contiguous K / V at every c, each layout of gpu_support.LAYOUTS at one of them; re-rotation wherever D % 16 == 0"""
    gen = torch.Generator(device=DEV).manual_seed(700 + D)
    B, H = 2, 2
    counts = [compaction_counts(ITEM_ROWS + c) for c in edge_counts(D // 8, SEL_U)]
    scores = mixed_scores((B, H, COMPACT_S), dtype, gen)
    inv = rope_inv_freq("theta1e4", D).to(DEV) if D % 16 == 0 else None
    k, v, kr = kv_for(B, H, COMPACT_S, D, dtype, gen)
    check_counts(scores, k, v, COMPACT_L, counts, f"compaction {_name(dtype)} D={D}", kr=kr, inv=inv)
    for i, kind in enumerate(LAYOUTS):
        k, v = (bits_of(t, gen) for t in _layout(kind, B, H, COMPACT_S, D, dtype, seed=D + i))
        kr = _layout(kind, B, H, COMPACT_S, D, dtype, seed=100 + D + i)[0]
        sc = scores[:, : k.shape[1]]
        check_counts(sc, k, v, COMPACT_L, [counts[i % len(counts)]], f"compaction {_name(dtype)} D={D} {kind}",
                     kr=kr, inv=inv)


# ---------------------------------------------------------------------------------------------------
# 6. entry-point contracts
# ---------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_name)
def test_fp32_scores_are_ranked_in_the_cache_dtype(dtype):
    """fp32 scores select as scores.to(cache dtype): in every chunk 1 + 2^-12 at offset 250 and 1 at offset 100 round to
    one tie, so chunk_kept = tail_kept = 1 keeps offset 100, where an fp32 ranking would keep 250"""
    gen = torch.Generator(device=DEV).manual_seed(800)
    B, H, L, S = 2, 2, 1000, 3500
    x = -torch.rand(B, H, S, generator=gen, device=DEV) - 1
    x[..., 100::L] = 1.0
    x[..., 250::L] = 1.0 + 2.0 ** -12
    r = x.to(dtype)
    assert torch.equal(r[..., 100::L], r[..., 250::L])
    k, v, kr = kv_for(B, H, S, 32, dtype, gen)
    inv = rope_inv_freq("theta1e4", 32).to(DEV)
    orders = chunk_orders(r, L)
    assert not torch.equal(chunked_canonical(x, L, 1, 1), chunked_from_orders(orders, L, 1, 1))
    check_counts(x, k, v, L, [(1, 1), (2, 2), (500, 250), (L, 500)], f"fp32 {_name(dtype)}", orders=orders, kr=kr,
                 inv=inv)
    assert torch.equal(call_chunked(x, k, v, L, 1, 1)[2][0, 0].long().cpu(), torch.arange(100, S, L))
    # the Python wrapper takes the same path
    out = native.scores_compress_chunked(x, k, v, 0.5, L, None, True)
    assert_idx(out[2], chunked_from_orders(orders, L, *native.chunk_counts(S, L, 0.5)[1:3]), "wrapper")


SCORE_STRIDES = ["every_other_head", "broadcast_over_b", "broadcast_over_h", "transposed"]


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_name)
@pytest.mark.parametrize("kind", SCORE_STRIDES)
def test_score_strides(kind, dtype):
    gen = torch.Generator(device=DEV).manual_seed(810 + SCORE_STRIDES.index(kind))
    B, H, S, L = 3, 4, 2333, 1000
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
    check_counts(scores, k, v, L, [(1, 333), (500, 1), (L, 333)], f"strides {kind} {_name(dtype)}", kr=kr, inv=inv)


WS_S = sorted({S for _, S in GEOMETRY} | {PS, COMPACT_S, 3000, 131072})


def _raw(p, scores, k, v, L, ck, tk, ws, nbytes):
    """kvp_scores_compress_chunked on the workspace `ws` (nbytes of it); (K', V', idx)"""
    sc, sstride = native._caller_scores(scores, k)
    n = p.n_kept
    B, H, _, D = k.shape
    outs = (torch.empty(B, H, n, D, device=DEV, dtype=k.dtype), torch.empty(B, H, n, D, device=DEV, dtype=k.dtype),
            torch.empty(B, H, n, device=DEV, dtype=torch.int32))
    native._enqueue("kvp_scores_compress_chunked", k.device, p, sc, sstride, L, ck, tk, k, v, None, *outs, ws, nbytes)
    return outs


def _accepts(p, scores, k, v, L, ck, tk, ws, nbytes) -> bool:
    try:
        _raw(p, scores, k, v, L, ck, tk, ws, nbytes)
    except RuntimeError as e:
        assert "workspace too small" in str(e), e
        return False
    return True


def smallest_workspace(p, scores, k, v, L, ck, tk, ws) -> int:
    """The smallest multiple of 256 bytes the call accepts, by bisection between 0 (refused: a refused call returns
    before it enqueues anything) and ws.numel() (accepted)"""
    lo, hi = 0, ws.numel() // 256
    assert not _accepts(p, scores, k, v, L, ck, tk, ws, 0) and _accepts(p, scores, k, v, L, ck, tk, ws, hi * 256)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if _accepts(p, scores, k, v, L, ck, tk, ws, mid * 256):
            hi = mid
        else:
            lo = mid
    return hi * 256


@gpu
def test_exact_size_and_smallest_workspaces():
    """A workspace of exactly kvp_workspace_bytes(KVP_SCORER_FINCH), filled with 0xFF, gives the usual result bitwise,
    and so does the smallest one the call accepts (the Finch layout at window 1); 256 bytes less is refused. The Finch
    size, sized for window S - 1, is at least that smallest size at every S of the case lists."""
    gen = torch.Generator(device=DEV).manual_seed(900)
    B, H, S, D, L = 2, 2, 3000, 64, 700
    scores = mixed_scores((B, H, S), torch.bfloat16, gen)
    k, v, kr = kv_for(B, H, S, D, torch.bfloat16, gen)
    ck, tk = 300, 100
    n = n_kept_of(S, L, ck, tk)
    p = native.make_problem(k, v, n)
    n_bytes = native.workspace_bytes(p, native.SCORER_FINCH)
    ws = torch.full((n_bytes,), 0xFF, dtype=torch.uint8, device=DEV)
    want = call_chunked(scores, k, v, L, ck, tk, check=True)
    _same_outputs(_raw(p, scores, k, v, L, ck, tk, ws, n_bytes), want, "exact size")
    small = smallest_workspace(p, scores, k, v, L, ck, tk, ws)
    ws.fill_(0xFF)
    _same_outputs(_raw(p, scores, k, v, L, ck, tk, ws, small), want, "smallest size")
    with pytest.raises(RuntimeError, match="workspace too small"):
        _raw(p, scores, k, v, L, ck, tk, ws, small - 256)
    assert small <= n_bytes
    for S in WS_S:
        sc = mixed_scores((1, 1, S), torch.bfloat16, gen)
        kk, vv, _ = kv_for(1, 1, S, 8, torch.bfloat16, gen)
        Lc = max(1, S // 3)
        ck, tk = 1, 1 if S % Lc else 0
        p = native.make_problem(kk, vv, n_kept_of(S, Lc, ck, tk))
        need = native.workspace_bytes(p, native.SCORER_FINCH)
        buf = torch.empty(need, dtype=torch.uint8, device=DEV)
        assert smallest_workspace(p, sc, kk, vv, Lc, ck, tk, buf) <= need, f"S={S}"
    torch.cuda.synchronize()


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_name)
def test_graph_replay_with_scores_updated_in_place(dtype):
    nat = _native()
    gen = torch.Generator(device=DEV).manual_seed(910)
    B, H, S, D, L, ck, tk = 2, 3, 9100, 32, 1000, 400, 37
    scores = mixed_scores((B, H, S), dtype, gen)
    k, v, kr = kv_for(B, H, S, D, dtype, gen)
    inv = rope_inv_freq("theta1e4", D).to(DEV)
    graphed = nat.capture(lambda: (*_chunked(scores, k, v, L, ck, tk), *_chunked(scores, kr, v, L, ck, tk, inv)))
    for seed in (911, 912):
        scores.copy_(mixed_scores((B, H, S), dtype, torch.Generator(device=DEV).manual_seed(seed)))
        k_out, v_out, idx, kr_out, vr_out, idx_r = graphed.replay()
        torch.cuda.synchronize()
        want = chunked_canonical(scores, L, ck, tk)
        assert_idx(idx, want, f"graph replay seed {seed}")
        assert_idx(idx_r, want, f"graph replay rerotate seed {seed}")
        assert_gather(k_out, k, want, "graph replay K'")
        assert_gather(v_out, v, want, "graph replay V'")
        assert_gather(vr_out, v, want, "graph replay rerotate V'")
        assert_rerotated(kr_out, kr, want, inv, "graph replay rerotate")
        _same_outputs(call_chunked(scores, k, v, L, ck, tk), (k_out, v_out, idx), "graph replay vs eager")
    _check_ws(k, v, n_kept_of(S, L, ck, tk))


@gpu
def test_two_streams_concurrently():
    """Large calls on two streams at once, each with its own cached workspace, equal the same calls run serially"""
    nat = _native()
    gen = torch.Generator(device=DEV).manual_seed(920)
    B, H, S, D, L, ck, tk = 2, 8, 100000, 16, 30000, 15000, 5000
    n = n_kept_of(S, L, ck, tk)
    inputs = []
    for _ in range(2):
        inputs.append((mixed_scores((B, H, S), torch.bfloat16, gen), *kv_for(B, H, S, D, torch.bfloat16, gen)[:2]))
    serial = [call_chunked(sc, k, v, L, ck, tk) for sc, k, v in inputs]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for s in streams:
        s.wait_stream(torch.cuda.current_stream())
    outs = []
    for _ in range(3):  # repeated, so the streams' calls overlap
        for s, (sc, k, v) in zip(streams, inputs):
            with torch.cuda.stream(s):
                outs.append(call_chunked(sc, k, v, L, ck, tk))
    torch.cuda.synchronize()
    workspaces = set()
    for s, (sc, k, v) in zip(streams, inputs):
        with torch.cuda.stream(s):
            _check_ws(k, v, n)
            p = nat.make_problem(k, v, n)
            workspaces.add(nat._workspace(p, nat.SCORER_FINCH, torch.device(DEV)).data_ptr())
    assert len(workspaces) == 2, "the two streams share a workspace"
    for i, out in enumerate(outs):
        _same_outputs(out, serial[i % 2], f"stream call {i}")
    for (sc, k, v), (k_out, v_out, idx) in zip(inputs, serial):
        want = chunked_canonical(sc, L, ck, tk)
        assert_idx(idx, want, "serial call")
        assert_gather(k_out, k, want, "serial call K'")
        assert_gather(v_out, v, want, "serial call V'")
