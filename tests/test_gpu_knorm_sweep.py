"""KnormPress compress on all three of its paths against a float64 reference, at every kernel instantiation, queue
regime, refine-group boundary, planted selection edge and cache layout.

`kvp_knorm_compress` runs one of three implementations, chosen from the shape by `knorm_path()` (api.cu):
  * cluster: `knorm_cluster_kernel<T, KPT>` (knorm_cluster.cu), one launch, when the row fits one thread-block cluster;
  * fused: memset + `knorm_fused_kernel<T, LPR>` (select_compact.cu), when K is at most 32 MiB;
  * two kernels: memset + `knorm_score_kernel<T, LPR>` + `select_compact_kernel<void>` otherwise.
`knorm_dispatch` below restates that choice; the CPU tests check it against `kvp_launches_per_compress` and check that
the sweep reaches every instantiation the sources build and every queue regime of the fused kernel. Each GPU case also
asserts the path it takes.

Bars (the helpers are those of tests/test_gpu_scorer_sweep.py):
  1. every score is within 1 ulp of -sqrt(sum k^2) evaluated in float64 on the device and rounded once, and rows with
     >= 500 normal-range positions have no mean relative bias beyond 8 standard errors of rounding noise. The keys are
     randn rows scaled log-uniformly over many binades, so the scores fill many high-byte bins of the selection. At
     head_dim 128 a dropped element moves a score by about 0.4 % on average, roughly one bf16 ulp: the 1-ulp bar alone
     may let it through, the bias bar does not;
  2. `idx` is the lowest-index-ties top-k of the kernel's own scores, and K' / V' are exact gathers;
  3. the fused and two-kernel compress scores are bitwise equal to `knorm_score` (both run `knorm_score_chunk`); the
     cluster kernel sums in another order, so its scores are within 1 ulp of it;
  4. planted rows x * e_j have the exact score -|x|: there the scores must be bitwise equal to `-k.norm(dim=-1)` on the
     device (the reference's formula, which also gives the special rows: zero, +-inf, NaN, fp16 norms past 65504, fp16
     subnormal norms, bf16 rows whose fp32 sum of squares overflows) and the selection must be the canonical one of
     those scores, independent of the kernel's own;
  5. strided layouts are consumed in place and give outputs bitwise equal to contiguous copies;
  6. the same inputs give bitwise-equal outputs on the fused and two-kernel paths, and 1-ulp-close scores with a
     canonical selection on the cluster path (`kvp_debug_knorm_first_path` sets the first path the dispatch may take);
  7. fused and two kernels: optional outputs do not change K' / V', two calls are bitwise equal, a captured call replays
     correctly on new inputs, and no bounded wait expires.
Measured on an H100 80GB HBM3 (700 W power limit) over every case of this file: at most 1 ulp from the rounded fp64
score on every path; at most 2e-4 of a case's positions at 1 ulp on the cluster path, 1e-4 on the fused path and below
5e-5 on two kernels; the worst row bias is 0.32 of its bound. Each bar is asserted as stated above, not at the measured
values.
"""
import json
import re
import subprocess
from collections import namedtuple
from pathlib import Path

import pytest
import torch

from oracle import press_oracle as O
from tests.conftest import ulp16_diff
from tests.abi_cases import PYTHON, child_env
from tests.gpu_support import (assert_compress, assert_vs_ref64, _bits, _gather, knorm_ref64, LANES_PER_ROW,
                               lanes_per_row, _layout, LAYOUTS, _name, _native, _same)

gpu = pytest.mark.gpu
DEV = "cuda:0"
ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "kvpress_b200" / "csrc"
DTYPES = [torch.bfloat16, torch.float16]
PATHS = ("cluster", "fused", "two_kernels")  # in dispatch order: kvp_debug_knorm_first_path's 0, 1, 2
PATH_OF_LAUNCHES = {1 + i: path for i, path in enumerate(PATHS)}


# ---------------------------------------------------------------------------------------------------
# the dispatch: knorm_path (api.cu), choose_cluster / cluster_plan / launch_knorm_cluster (knorm_cluster.cu),
# launch_knorm_fused_t (select_compact.cu), launch_knorm_t (knorm.cu)
# ---------------------------------------------------------------------------------------------------
CL_THREADS, CL_MAX_KPT, CL_MAX_SMEM = 256, 24, 200 * 1024
FUSED_MAX_BYTES = 32 << 20  # K bytes up to which the fused kernel runs
BIG_ROW_BYTES = 8 << 20  # one kv-head row of K from which the fused queue runs at lag 1
REFINE_SPAN = 16 * 256  # positions of one refine item: 16 tiles of 256

Dispatch = namedtuple("Dispatch", "path dtype inst C v_smem lag R")  # inst: KPT (cluster) or LPR (fused, two kernels)


def cluster_plan(S: int, D: int, C: int):
    """(positions per CTA, v_smem, fits) of cluster_plan()."""
    P = ((S + C - 1) // C + 7) // 8 * 8
    tile, keys, lst = P * 2 * D, C * P * 2, P * 4
    v_smem = int(2 * tile + keys + lst + 64 <= CL_MAX_SMEM)
    smem = (2 if v_smem else 1) * tile + keys + lst + 64
    return P, v_smem, smem <= CL_MAX_SMEM and S <= CL_THREADS * CL_MAX_KPT


def cluster_size(S: int) -> int:
    C = 8
    while C > 1 and (S + C - 1) // C < 64:
        C >>= 1
    return C


def knorm_dispatch(B: int, H: int, S: int, D: int, dtype) -> Dispatch:
    R, name = B * H, _name(dtype)
    C = cluster_size(S)
    _, v_smem, fits = cluster_plan(S, D, C)
    if fits and R <= 65535:
        return Dispatch("cluster", name, 12 if S <= CL_THREADS * 12 else CL_MAX_KPT, C, v_smem, None, R)
    if B * H * S * D * 2 <= FUSED_MAX_BYTES:
        lag = 1 if S * D * 2 >= BIG_ROW_BYTES else 2
        return Dispatch("fused", name, lanes_per_row(D), None, None, min(lag, R), R)
    return Dispatch("two_kernels", name, lanes_per_row(D), None, None, None, R)


# ---------------------------------------------------------------------------------------------------
# the cases: (path each must take, (B, H, S, D))
# ---------------------------------------------------------------------------------------------------
SHAPES = [
    # fused, lag 2
    ("fused", (1, 8, 5889, 128)),  # first S past the cluster's shared-memory bound
    ("fused", (1, 8, 16384, 128)),  # exactly 32 MiB of K: a Llama-3.1-8B layer at 16k
    ("fused", (4, 8, 8192, 64)),
    ("fused", (1, 32, 8192, 32)),
    ("fused", (1, 8, 10000, 96)),  # LPR 16 with 12 pieces per row: a partial sub-warp
    ("fused", (1, 8, 3073, 256)),
    ("fused", (2, 3, 7000, 136)),  # LPR 32, 17 pieces per row
    # fused, lag 1: rows of 8 MiB and more, K loads evict_last
    ("fused", (1, 4, 32768, 128)),
    ("fused", (2, 1, 32768, 128)),
    ("fused", (1, 2, 16384, 256)),
    ("fused", (1, 4, 65536, 64)),
    ("fused", (1, 2, 131072, 32)),
    ("fused", (1, 1, 8000, 24)),  # lag clipped to R = 1
    # fused, S on both sides of a refine-group boundary
    *[("fused", (1, 8, S, 256)) for S in (4095, 4096, 4097)],
    *[("fused", (1, 8, S, 128)) for S in (8191, 8192, 8193)],
    # two kernels
    ("two_kernels", (1, 8, 16385, 128)),  # one position past 32 MiB
    ("two_kernels", (8, 8, 8192, 64)),
    ("two_kernels", (4, 32, 8192, 32)),
    ("two_kernels", (1, 8, 12000, 256)),
    ("two_kernels", (3, 8, 9000, 200)),
    ("two_kernels", (16, 8, 6145, 64)),  # R = 128
    *[("two_kernels", (8, 8, S, 256)) for S in (4095, 4096, 4097)],
    *[("two_kernels", (32, 8, S, 128)) for S in (8191, 8192, 8193)],
    # cluster
    ("cluster", (1, 8, 5888, 128)),  # the largest S at head_dim 128
    ("cluster", (1, 8, 3072, 256)),  # the largest S at head_dim 256
    ("cluster", (1, 4, 3072, 128)),  # KPT 12, V staged in shared memory
    ("cluster", (1, 4, 3073, 128)),  # KPT 24, V through registers
    *[("cluster", (2, 3, S, 128)) for S in (60, 100, 200, 300)],  # clusters of 1, 1, 2 and 4 CTAs
]
SWEEP = [(path, shape, dt) for path, shape in SHAPES for dt in DTYPES]

# planted scores: one shape per path, S past a refine-group boundary
PLANT_SHAPES = {"cluster": (2, 4, 5000, 128), "fused": (2, 4, 8200, 128), "two_kernels": (2, 8, 9000, 128)}
PLANT_KINDS = ["all_equal", "two_values", "threshold_key_lo00", "threshold_key_loff", "ties_across_refine_groups",
               "ties_across_cluster_slices", "zero_rows", "inf_rows", "nan_rows", "fp16_norm_overflow",
               "fp16_subnormal_norms", "bf16_sum_of_squares_overflow"]
PLANTED = [(path, kind, dt) for path in PLANT_SHAPES for kind in PLANT_KINDS for dt in DTYPES
           if not (kind.startswith("fp16") and dt != torch.float16) and not (kind.startswith("bf16") and dt != torch.bfloat16)]

# layouts: (B, H, S, D) per path; H = 1 for one_head_of_wider_cache
LAYOUT_SHAPES = {"cluster_v_smem1": (3, 4, 1500, 128), "cluster_v_smem0": (3, 4, 5000, 128),
                 "fused": (3, 4, 6000, 128), "two_kernels": (3, 4, 12000, 128)}
LAYOUT_S_H1 = {"cluster_v_smem1": 1500, "cluster_v_smem0": 5000, "fused": 6000, "two_kernels": 45000}


def layout_shape(where: str, kind: str):
    B, H, S, D = LAYOUT_SHAPES[where]
    return (B, 1, LAYOUT_S_H1[where], D) if kind == "one_head_of_wider_cache" else (B, H, S, D)


LAYOUT_CASES = [(where, kind, dt) for where in LAYOUT_SHAPES for kind in LAYOUTS for dt in DTYPES]

CROSS_SHAPES = [(1, 8, 2560, 128), (2, 4, 5000, 64)]
CALL_SHAPES = {"fused": (2, 4, 6000, 128), "two_kernels": (3, 4, 12000, 128)}


def _all_cases():
    """(path, (B, H, S, D)) of every GPU case of this file."""
    out = [(p, s) for p, s, _ in SWEEP] + [(p, PLANT_SHAPES[p]) for p in PLANT_SHAPES]
    out += [("cluster" if w.startswith("cluster") else w, layout_shape(w, kind)) for w in LAYOUT_SHAPES for kind in LAYOUTS]
    out += list(CALL_SHAPES.items()) + [("cluster", s) for s in CROSS_SHAPES]
    return out


# ---------------------------------------------------------------------------------------------------
# CPU: the restated dispatch agrees with the library, and the sweep reaches every instantiation and regime
# ---------------------------------------------------------------------------------------------------
_LAUNCHES_CHILD = r"""
import ctypes, importlib.util, json, sys
spec = importlib.util.spec_from_file_location("kvp_native", sys.argv[1])
nat = importlib.util.module_from_spec(spec)
spec.loader.exec_module(nat)
lib = nat.load()


def launches():
    out = []
    for B, H, S, D in json.loads(sys.argv[2]):
        p = nat.KvpProblem()
        p.B, p.Hkv, p.Hq, p.S, p.D, p.n_kept, p.dtype = B, H, H, S, D, 1, 0
        p.k_stride = p.v_stride = (ctypes.c_int64 * 3)(H * S * D, S * D, D)
        out.append(nat.launches_per_compress(p, nat.SCORER_KNORM))
    return out


res = {"default": launches(), "previous": []}
for first in (1, 2, 0):
    res["previous"].append(lib.kvp_debug_knorm_first_path(first))
    res[str(first)] = launches()
res["rejected"] = [lib.kvp_debug_knorm_first_path(first) for first in (-1, 3)]
res["after_rejected"] = launches()
print(json.dumps(res))
"""


def test_knorm_dispatch_matches_launch_count():
    """kvp_launches_per_compress (1 = cluster, 2 = fused, 3 = two kernels) agrees with knorm_dispatch on every case
    shape, and every case is listed under the path knorm_dispatch gives it. kvp_debug_knorm_first_path(1 or 2) moves
    every case to the path it forces, or to two kernels where K is too large for the fused kernel; the hook returns
    the previous value, rejects values outside 0..2 and, set back to 0, restores the default dispatch. No device: a
    child process that sees none."""
    cases = sorted(set(_all_cases()))
    for path, shape in cases:
        assert knorm_dispatch(*shape, torch.bfloat16).path == path, (path, shape)
    shapes = [s for _, s in cases]
    r = subprocess.run([*PYTHON, "-c", _LAUNCHES_CHILD, str(ROOT / "kvpress_b200" / "native.py"), json.dumps(shapes)],
                       cwd=ROOT, env=child_env(CUDA_VISIBLE_DEVICES=""), capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-4000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    assert got["previous"] == [0, 1, 2] and got["rejected"] == [-1, -1]
    assert got["0"] == got["default"] and got["after_rejected"] == got["default"]
    for first in ("default", "1", "2"):
        forced = 0 if first == "default" else int(first)
        want = [PATHS[max(PATHS.index(path), forced)] for path, _ in cases]
        wrong = [(shape, PATH_OF_LAUNCHES[n], w) for (_, shape), n, w in zip(cases, got[first], want)
                 if PATH_OF_LAUNCHES[n] != w]
        assert not wrong, f"first path {first}: (shape, library path, restated path): {wrong}"


def test_lanes_per_row_follows_common():
    """lanes_per_row restates with_lanes_per_row over kLanesPerRow: ascending power-of-two lane counts of one warp, the
    last covering the widest head_dim (256); every head_dim takes the first count >= D / 8 and each count is taken."""
    assert LANES_PER_ROW == (4, 8, 16, 32)  # the instantiations the sweeps' head_dims are chosen for
    assert 8 * LANES_PER_ROW[-1] >= 256
    for D in range(8, 257, 8):
        assert lanes_per_row(D) == min(lpr for lpr in LANES_PER_ROW if D // 8 <= lpr)
    assert {lanes_per_row(D) for D in range(8, 257, 8)} == set(LANES_PER_ROW)


def _built_instantiations():
    """{(path, dtype, LPR or KPT)} the sources instantiate."""
    cl_src = (CSRC / "knorm_cluster.cu").read_text()
    max_kpt = re.search(r"constexpr int kClMaxKeysPerThread = (\d+);", cl_src).group(1)
    cluster = re.findall(r"launch_cluster_t<T, (12|kClMaxKeysPerThread)>\(", cl_src)  # T: both, through with_dtype
    assert int(max_kpt) == CL_MAX_KPT
    built = {(path, n, lpr) for path in ("fused", "two_kernels") for n in ("bf16", "fp16") for lpr in LANES_PER_ROW}
    built |= {("cluster", n, int(max_kpt if k == "kClMaxKeysPerThread" else k)) for k in cluster for n in ("bf16", "fp16")}
    return built


def test_knorm_sweep_reaches_every_dispatched_instantiation_and_regime():
    """The shape sweep runs every <T, LPR> of the fused and score kernels and every <T, KPT> of the cluster kernel, the
    fused queue at lag 2, at lag 1 with R >= 2 and at lag 1 clipped to R = 1, and the cluster kernel with 1, 2, 4 and 8
    CTAs, with and without V staged in shared memory."""
    built = _built_instantiations()
    assert len(built) == 20
    got = [knorm_dispatch(*shape, dt) for _, shape, dt in SWEEP]
    assert {(d.path, d.dtype, d.inst) for d in got} == built
    fused = [d for d in got if d.path == "fused"]
    assert any(d.lag == 2 for d in fused)
    assert any(d.lag == 1 and d.R >= 2 for d in fused)
    assert any(d.lag == 1 and d.R == 1 for d in fused)
    cl = [d for d in got if d.path == "cluster"]
    assert {d.C for d in cl} == {1, 2, 4, 8} and {d.v_smem for d in cl} == {0, 1}
    # the layout cases stage V in shared memory and leave it in global memory (the strided-V bulk copies)
    assert {knorm_dispatch(*layout_shape(w, "transposed_bshd"), torch.bfloat16).v_smem
            for w in ("cluster_v_smem0", "cluster_v_smem1")} == {0, 1}
    # the planted ties straddle a refine-group boundary on every path
    assert all(s[2] > REFINE_SPAN + 8 for s in PLANT_SHAPES.values())


# ---------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------


def sweep_inputs(B, H, S, D, dtype, seed):
    """randn keys, each row scaled by 2^u with u uniform over many binades (fp16 norms stay normal and finite)."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    lo, hi = (-20.0, 20.0) if dtype == torch.bfloat16 else (-10.0, 8.0)
    scale = torch.exp2(torch.rand(B, H, S, 1, generator=gen, device=DEV) * (hi - lo) + lo)
    k = (torch.randn(B, H, S, D, generator=gen, device=DEV) * scale).to(dtype)
    v = torch.randn(B, H, S, D, generator=gen, device=DEV).to(dtype)
    return k, v


def n_kept_values(S: int):
    return sorted({n for n in (1, 256, 257, S // 2, S - 1, S) if 1 <= n <= S})


def _path(nat, k, v) -> str:
    return PATH_OF_LAUNCHES[nat.launches_per_compress(nat.make_problem(k, v, 1), nat.SCORER_KNORM)]


def _check_workspace(nat, k, v, n_kept):
    p = nat.make_problem(k, v, n_kept)
    nat.workspace_check(p, nat.SCORER_KNORM, nat._workspace(p, nat.SCORER_KNORM, k.device))


def run_knorm(k, v, path, what, n_kept_list=None):
    """Bars 1-3 for one problem: every n_kept of the list, scores against fp64 once and equal across the calls."""
    nat = _native()
    S = k.shape[2]
    assert _path(nat, k, v) == path, what
    ref = knorm_ref64(k)
    stats, first = None, None
    for n in n_kept_list or n_kept_values(S):
        k_out, v_out, idx, sc = nat.knorm_compress(k, v, n, return_indices=True, return_scores=True)
        if path != "cluster":
            _check_workspace(nat, k, v, n)
        if first is None:
            first = sc
            stats = assert_vs_ref64(sc, ref, torch.zeros(S, dtype=torch.bool), what)
        else:
            assert _same(sc, first), f"{what}: scores depend on n_kept"
        assert_compress(k, v, k_out, v_out, idx, sc, n)
    alone = nat.knorm_score(k)
    if path == "cluster":
        assert ulp16_diff(first, alone).max() <= 1, f"{what}: cluster scores beyond 1 ulp of knorm_score"
    else:
        assert _same(first, alone), f"{what}: compress scores differ from knorm_score"
    return stats


# ---------------------------------------------------------------------------------------------------
# 1. the shape sweep
# ---------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("path,shape,dtype", SWEEP,
                         ids=[f"{p}-{_name(dt)}-b{s[0]}h{s[1]}s{s[2]}d{s[3]}" for p, s, dt in SWEEP])
def test_knorm_sweep(path, shape, dtype):
    d = knorm_dispatch(*shape, dtype)
    B, H, S, D = shape
    k, v = sweep_inputs(B, H, S, D, dtype, S * 131 + D * 7 + B * 3 + H)
    run_knorm(k, v, path, f"knorm {path} {_name(dtype)} {shape} inst={d.inst} C={d.C} v_smem={d.v_smem} lag={d.lag}")


# ---------------------------------------------------------------------------------------------------
# 2. planted scores and special rows
# ---------------------------------------------------------------------------------------------------
def _one_bits(dtype) -> int:
    return 0x3F80 if dtype == torch.bfloat16 else 0x3C00  # 1.0


def _randbits(lo, hi, shape, gen):
    return torch.randint(lo, hi + 1, shape, generator=gen, device=DEV)


def _rank(shape, gen):
    """a random permutation of the positions of every row"""
    return torch.rand(*shape, generator=gen, device=DEV).argsort(-1)


def planted(path, kind, dtype, seed):
    """(k, n_kept values, mask of the rows planted as x * e_j) of one planted case. Every (b, h) row holds the same
    multiset of scores in its own order, so that one n_kept puts the threshold where the case wants it in every row."""
    B, H, S, D = PLANT_SHAPES[path]
    gen = torch.Generator(device=DEV).manual_seed(seed)
    one = _one_bits(dtype)
    shape = (B, H, S)
    mag = _randbits(one - 600, one + 600, shape, gen)  # |score| bits: a smaller magnitude is a larger score
    rank = _rank(shape, gen)
    n_list = n_kept_values(S)
    special = None  # rows that are not x * e_j: (mask, row value [D])

    def put(lo, hi, bits):  # the positions of rank [lo, hi) in every row get `bits` (a tensor or an int)
        pos = rank[..., lo:hi]
        mag.scatter_(2, pos, bits if torch.is_tensor(bits) else torch.full_like(pos, bits))

    def rows(lo, hi):
        m = torch.zeros(shape, dtype=torch.bool, device=DEV)
        m.scatter_(2, rank[..., lo:hi], True)
        return m

    if kind == "all_equal":
        mag.fill_(one + 64)
    elif kind == "two_values":
        put(0, S // 3, one)
        put(S // 3, S, one + 128)
        n_list += [S // 3]
    elif kind.startswith("threshold_key"):
        # ordered key of -|x| = 0x7FFF - bits(|x|): low byte 0x00 <=> bits(|x|) & 0xFF == 0xFF, 0xFF <=> == 0x00. The
        # keys next to the threshold's then fall into the neighbouring high-byte bin, and many positions hold them.
        mt = 0x3FFF if kind.endswith("lo00") else 0x4000
        n_gt, n_eq = S // 3, 50
        put(0, n_gt // 2, mt - 1)
        put(n_gt // 2, n_gt, _randbits(mt - 300, mt - 2, (B, H, n_gt - n_gt // 2), gen))
        put(n_gt, n_gt + n_eq, mt)
        mid = n_gt + n_eq + (S - n_gt - n_eq) // 2
        put(n_gt + n_eq, mid, mt + 1)
        put(mid, S, _randbits(mt + 2, mt + 300, (B, H, S - mid), gen))
        n_list = [n_gt - 1, n_gt, n_gt + 1, n_gt + 25, n_gt + n_eq, n_gt + n_eq + 1]
    elif kind.startswith("ties_across"):
        # 16 tied positions around a refine-group boundary, or a cluster slice boundary (a 256-position tile boundary
        # off the cluster path); half of the other positions score above the ties, half below
        if kind == "ties_across_refine_groups":
            c = REFINE_SPAN
        else:
            c = 2 * cluster_plan(S, D, cluster_size(S))[0] if path == "cluster" else 1280
        tie = torch.arange(c - 8, c + 8, device=DEV)
        rest = torch.cat([torch.arange(0, c - 8, device=DEV), torch.arange(c + 8, S, device=DEV)])
        order = rest[_rank((B, H, rest.numel()), gen)]
        n_gt = rest.numel() // 2
        mag.scatter_(2, order[..., :n_gt], _randbits(one - 600, one - 1, (B, H, n_gt), gen))
        mag.scatter_(2, order[..., n_gt:], _randbits(one + 1, one + 600, (B, H, rest.numel() - n_gt), gen))
        mag[..., tie] = one
        n_list = [n_gt + 7, n_gt + 8, n_gt + 9]
    elif kind == "zero_rows":  # -0, the largest score a norm can give; the selection orders it as 0
        z = S // 10
        put(0, z, 0)
        n_list += [z - 1, z, z + 1]
    elif kind == "inf_rows":  # +-inf: -inf
        n = S // 20
        put(0, n, 0x7F80 if dtype == torch.bfloat16 else 0x7C00)
        n_list += [S - n - 1, S - n, S - n + 1]
    elif kind == "nan_rows":  # NaN, the largest key: kept first, ties to the lowest positions
        n = S // 30
        put(0, n, 0x7FC0 if dtype == torch.bfloat16 else 0x7E00)
        n_list += [n - 1, n, n + 1]
    elif kind == "fp16_norm_overflow":  # all elements 6000: the norm 67882 rounds to inf; and single 65504s
        n = S // 20
        put(n, 2 * n, 0x7BFF)
        special = (rows(0, n), torch.full((D,), 6000.0))
        n_list += [S - n - 1, S - n, S - n + 1]
    elif kind == "fp16_subnormal_norms":  # subnormal magnitudes and the smallest normals
        mag.copy_(_randbits(1, 0x0500, shape, gen))
    elif kind == "bf16_sum_of_squares_overflow":  # four elements 2^64: the fp32 sum of squares overflows; single 2^63s
        n = S // 20
        put(n, 2 * n, 0x5F00)
        row = torch.zeros(D)
        row[:4] = 2.0 ** 64
        special = (rows(0, n), row)
        n_list += [S - n - 1, S - n, S - n + 1]
    x = mag.to(torch.int16).view(dtype)
    x = torch.where(torch.rand(shape, generator=gen, device=DEV) < 0.5, x, -x)  # the sign does not change the norm
    j = (torch.arange(S, device=DEV) % D).expand(B, H, S)
    k = torch.zeros(B, H, S, D, dtype=dtype, device=DEV)
    k.scatter_(3, j.unsqueeze(-1), x.unsqueeze(-1))
    plain = torch.ones(shape, dtype=torch.bool, device=DEV)
    if special is not None:
        mask, row = special
        k[mask] = row.to(dtype=dtype, device=DEV)
        plain &= ~mask
    v = torch.randn(B, H, S, D, generator=gen, device=DEV).to(dtype)
    return k, v, sorted({n for n in n_list if 1 <= n <= S}), plain, mag


@gpu
@pytest.mark.parametrize("path,kind,dtype", PLANTED, ids=[f"{p}-{k}-{_name(dt)}" for p, k, dt in PLANTED])
def test_knorm_planted_scores(path, kind, dtype):
    nat = _native()
    k, v, n_list, plain, mag = planted(path, kind, dtype, 17 + PLANT_KINDS.index(kind))
    assert _path(nat, k, v) == path
    want = -k.norm(dim=-1)  # the reference's formula (knorm_press.py:38), also for the special rows
    # the planted rows score exactly -|x|
    finite = plain & (mag < (0x7F80 if dtype == torch.bfloat16 else 0x7C00))
    assert torch.equal(_bits(want)[finite], (mag | 0x8000).to(torch.int16)[finite])
    nan = torch.isnan(want)
    want_idx = {n: O.select_lowest_index_ties(want.cpu(), n) for n in n_list}
    for n in n_list:
        k_out, v_out, idx, sc = nat.knorm_compress(k, v, n, return_indices=True, return_scores=True)
        if path != "cluster":
            _check_workspace(nat, k, v, n)
        assert torch.equal(torch.isnan(sc), nan), f"{kind} n_kept={n}: NaN scores differ"
        assert torch.equal(_bits(sc)[~nan], _bits(want)[~nan]), \
            f"{kind} n_kept={n}: {int((_bits(sc)[~nan] != _bits(want)[~nan]).sum())} scores differ from -k.norm"
        assert torch.equal(idx.long().cpu(), want_idx[n]), f"{kind} n_kept={n}: not the canonical selection"
        # gathers compared bitwise: the kept NaN rows are not equal to themselves
        assert _same(k_out, _gather(k, idx)) and _same(v_out, _gather(v, idx)), f"{kind} n_kept={n}: not exact gathers"


# ---------------------------------------------------------------------------------------------------
# 3. strided layouts
# ---------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("where,kind,dtype", LAYOUT_CASES, ids=[f"{w}-{k}-{_name(dt)}" for w, k, dt in LAYOUT_CASES])
def test_knorm_strided_layouts(where, kind, dtype):
    nat = _native()
    B, H, S, D = layout_shape(where, kind)
    path = "cluster" if where.startswith("cluster") else where
    k, v = _layout(kind, B, H, S, D, dtype, 900 + S + D)
    assert nat._rows_ok(k) and nat._rows_ok(v) and not v.is_contiguous()
    if kind != "v_strided_k_contiguous":
        assert not k.is_contiguous()
    if where.startswith("cluster"):
        assert knorm_dispatch(B, H, S, D, dtype).v_smem == int(where[-1])
    kc, vc = k.contiguous(), v.contiguous()
    assert _path(nat, k, v) == path
    n_kept = O.kept_count(S, 0.4)
    got = nat.knorm_compress(k, v, n_kept, return_indices=True, return_scores=True)
    want = nat.knorm_compress(kc, vc, n_kept, return_indices=True, return_scores=True)
    assert all(_same(a, b) for a, b in zip(got, want)), f"{where} {kind}: differs from contiguous copies"
    assert_vs_ref64(got[3], knorm_ref64(kc), torch.zeros(S, dtype=torch.bool), f"knorm layout {where} {kind}")
    assert_compress(kc, vc, *got, n_kept)
    assert _same(nat.knorm_score(k), nat.knorm_score(kc))


# ---------------------------------------------------------------------------------------------------
# 4. the three paths on the same inputs (kvp_debug_knorm_first_path moves the cluster-sized cases off the cluster path)
# ---------------------------------------------------------------------------------------------------
def _run_cross(nat, launches):
    """{case: [k, v, k_out, v_out, idx, scores]} of every CROSS_SHAPES input on the path that takes `launches`."""
    res = {}
    for dt in DTYPES:
        for B, H, S, D in CROSS_SHAPES:
            gen = torch.Generator(device=DEV).manual_seed(S * 31 + D)
            scale = torch.exp2(torch.rand(B, H, S, 1, generator=gen, device=DEV) * 16 - 8)
            k = (torch.randn(B, H, S, D, generator=gen, device=DEV) * scale).to(dt)
            v = torch.randn(B, H, S, D, generator=gen, device=DEV).to(dt)
            for n in (257, S // 2):
                assert nat.launches_per_compress(nat.make_problem(k, v, n), nat.SCORER_KNORM) == launches
                out = nat.knorm_compress(k, v, n, return_indices=True, return_scores=True)
                res[f"{dt}-{B}x{H}x{S}x{D}-{n}"] = [k, v, *out]
    return res


@gpu
def test_knorm_paths_agree_on_one_input_through_the_first_path_hook():
    nat = _native()
    lib = nat.load()
    got = {}
    for first, path in enumerate(PATHS):
        previous = lib.kvp_debug_knorm_first_path(first)
        try:
            got[path] = _run_cross(nat, first + 1)
        finally:
            lib.kvp_debug_knorm_first_path(previous)
    assert len(got["cluster"]) == 2 * 2 * len(CROSS_SHAPES)
    for case, (k, v, k_out, v_out, idx, sc) in got["fused"].items():
        assert all(_same(a, b) for a, b in zip(got["cluster"][case][:2], (k, v))), f"{case}: inputs differ"
        assert all(_same(a, b) for a, b in zip(got["two_kernels"][case], (k, v, k_out, v_out, idx, sc))), \
            f"{case}: fused and two kernels differ"
        ck, cv, ck_out, cv_out, cidx, csc = got["cluster"][case]
        assert ulp16_diff(csc, sc).max() <= 1, f"{case}: cluster scores beyond 1 ulp of the fused ones"
        assert_compress(ck, cv, ck_out, cv_out, cidx, csc, cidx.shape[-1])
        assert_compress(k, v, k_out, v_out, idx, sc, idx.shape[-1])


# ---------------------------------------------------------------------------------------------------
# 5. call behaviour on the fused and two-kernel paths
# ---------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("path", list(CALL_SHAPES))
def test_knorm_call_behaviour(path, dtype):
    nat = _native()
    B, H, S, D = CALL_SHAPES[path]
    n = O.kept_count(S, 0.5)
    k, v = sweep_inputs(B, H, S, D, dtype, 1300 + S)
    assert _path(nat, k, v) == path

    def call(kk, vv, ri=True, rs=True):
        out = nat.knorm_compress(kk, vv, n, return_indices=ri, return_scores=rs)
        _check_workspace(nat, kk, vv, n)
        return out

    full = call(k, v)
    assert_compress(k, v, *full, n)
    # the optional outputs change nothing else; a second call is bitwise equal (the only atomics are integer counts)
    for ri, rs in ((False, False), (True, False), (False, True), (True, True)):
        out = call(k, v, ri, rs)
        assert _same(out[0], full[0]) and _same(out[1], full[1]), (ri, rs)
        assert _same(out[2], full[2] if ri else None) and _same(out[3], full[3] if rs else None), (ri, rs)
    # a captured call (memset node; on two kernels also the programmatic-dependent-launch edge) replayed on new inputs
    kk, vv = k.clone(), v.clone()
    graphed = nat.capture(lambda: nat.knorm_compress(kk, vv, n, return_indices=True, return_scores=True))
    k2, v2 = sweep_inputs(B, H, S, D, dtype, 1301 + S)
    kk.copy_(k2)
    vv.copy_(v2)
    replayed = [t.clone() for t in graphed.replay()]
    torch.cuda.synchronize()
    eager = call(kk, vv)
    assert all(_same(a, b) for a, b in zip(replayed, eager)), f"{path}: graph replay differs from an eager call"
    assert_compress(k2, v2, *replayed, n)
