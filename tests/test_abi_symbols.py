"""The C-ABI library loads on a machine without a GPU and exports every symbol include/kvpress_b200.h
declares (no compute calls here); argument validation paths that need no device are exercised too."""
import ctypes
import re
from pathlib import Path

import pytest

from kvpress_b200 import native

HEADER = Path(__file__).resolve().parent.parent / "include" / "kvpress_b200.h"


def declared_symbols():
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    return sorted(set(re.findall(r"\b(kvp_[a-z_0-9]+)\s*\(", text)))


def test_every_declared_symbol_is_exported_and_bound():
    lib = native.load()
    names = declared_symbols()
    assert len(names) >= 16
    for name in names:
        assert hasattr(lib, name), f"{name} declared in the header but not exported"
        assert name in native.SIGNATURES, f"{name} has no ctypes signature in native.py"
    assert sorted(native.SIGNATURES) == names


def test_status_strings_and_validation_without_gpu():
    lib = native.load()
    assert lib.kvp_abi_version() == 1
    assert lib.kvp_status_string(0) == b"ok"
    assert b"workspace" in lib.kvp_status_string(-5)
    p = native.KvpProblem()
    p.B, p.Hkv, p.Hq, p.S, p.D, p.n_kept, p.dtype = 1, 8, 32, 131072, 128, 39321, 0
    out = ctypes.c_size_t(0)
    assert lib.kvp_workspace_bytes(ctypes.byref(p), native.SCORER_KNORM, ctypes.byref(out)) == 0
    knorm_ws = out.value
    assert 2 * 8 * 131072 <= knorm_ws < 64 << 20
    assert lib.kvp_workspace_bytes(ctypes.byref(p), native.SCORER_EXPECTED_ATTENTION, ctypes.byref(out)) == 0
    assert out.value > knorm_ws
    p.D = 12
    assert lib.kvp_workspace_bytes(ctypes.byref(p), native.SCORER_KNORM, ctypes.byref(out)) == -2
    p.D, p.dtype = 128, 7
    assert lib.kvp_workspace_bytes(ctypes.byref(p), native.SCORER_KNORM, ctypes.byref(out)) == -3
    assert lib.kvp_workspace_bytes(None, native.SCORER_KNORM, ctypes.byref(out)) == -1
    n = ctypes.c_int(0)
    p.dtype = 0
    assert lib.kvp_launches_per_compress(ctypes.byref(p), native.SCORER_STREAMING, ctypes.byref(n)) == 0 and n.value == 1


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    monkeypatch.setattr(native, "_lib", None)
    monkeypatch.setenv("KVPRESS_B200_LIB", str(tmp_path / "nope.so"))
    with pytest.raises(native.NativeLibraryError, match="no CPU or PyTorch fallback"):
        native.load()


def test_argument_validation_of_every_compress_entry_point_without_gpu():
    """Error behaviour of the C ABI (include/kvpress_b200.h "Return value"): every check below fails before the first
    CUDA call, so it runs on the GPU-less build box. Pointers are fake, aligned, never dereferenced."""
    lib = native.load()
    P = ctypes.c_void_p
    good, odd = P(0x10000), P(0x10008 + 4)          # 16-byte aligned / misaligned
    stream = P(0)

    def problem(**kw):
        p = native.KvpProblem()
        p.B, p.Hkv, p.Hq, p.S, p.D, p.n_kept, p.dtype = 1, 2, 2, 1000, 128, 500, 0
        p.k_stride = (ctypes.c_int64 * 3)(2 * 1000 * 128, 1000 * 128, 128)
        p.v_stride = (ctypes.c_int64 * 3)(2 * 1000 * 128, 1000 * 128, 128)
        for k, v in kw.items():
            setattr(p, k, v)
        return p

    sstride = (ctypes.c_int64 * 2)(2000, 1000)
    calls = {
        "knorm": lambda p, K, ws, n: lib.kvp_knorm_compress(ctypes.byref(p), K, good, good, good, None, None, ws, n, stream),
        "keydiff": lambda p, K, ws, n: lib.kvp_keydiff_compress(ctypes.byref(p), K, good, good, good, None, None, ws, n, stream),
        "snapkv": lambda p, K, ws, n: lib.kvp_snapkv_compress(ctypes.byref(p), K, good, good, 64, 5, good, good, None, None, ws, n, stream),
        "expected_attention": lambda p, K, ws, n: lib.kvp_expected_attention_compress(
            ctypes.byref(p), K, good, good, good, 0.0, 4, 1, good, good, None, None, ws, n, stream),
        "generic": lambda p, K, ws, n: lib.kvp_scores_compress(ctypes.byref(p), good, sstride, K, good, good, good, None, ws, n, stream),
        "rerotate": lambda p, K, ws, n: lib.kvp_scores_compress_rerotate(
            ctypes.byref(p), good, sstride, K, good, ctypes.cast(good, ctypes.POINTER(ctypes.c_float)), good, good, None, ws, n, stream),
    }
    for name, call in calls.items():
        assert call(problem(), P(0), good, 1 << 30) == -1, name                  # NULL K
        assert call(problem(), odd, good, 1 << 30) == -4, name                   # misaligned K
        assert call(problem(n_kept=1001), good, good, 1 << 30) == -7, name        # n_kept > S
        assert call(problem(D=12), good, good, 1 << 30) == -2, name               # head_dim not a multiple of 8
        assert call(problem(dtype=3), good, good, 1 << 30) == -3, name            # unknown dtype
        bad = problem()
        bad.k_stride = (ctypes.c_int64 * 3)(2 * 1000 * 128, 1000 * 128, 100)     # rows overlap
        assert call(bad, good, good, 1 << 30) == -4, name
        assert call(problem(), good, good, 64) == -5, name                        # workspace too small
        assert call(problem(), good, P(0), 1 << 30) == -1, name                   # NULL workspace
        assert call(problem(n_kept=0), good, good, 1 << 30) == 0, name            # nothing to keep: no work, OK
    # streaming has no workspace; selection-only has no K/V
    p = problem()
    assert lib.kvp_streaming_compress(ctypes.byref(p), 4, P(0), good, good, good, None, stream) == -1
    assert lib.kvp_scores_select(ctypes.byref(p), P(0), sstride, ctypes.cast(good, ctypes.POINTER(ctypes.c_int32)), good,
                                 1 << 30, stream) == -1
    assert lib.kvp_scores_select(ctypes.byref(p), good, sstride, None, good, 1 << 30, stream) == -1
    assert lib.kvp_scores_select(ctypes.byref(p), good, sstride, ctypes.cast(good, ctypes.POINTER(ctypes.c_int32)), good,
                                 64, stream) == -5
    # workspace sizing is monotone in S and covers every scorer id
    sizes = []
    for scorer in range(6):
        out = ctypes.c_size_t(0)
        assert lib.kvp_workspace_bytes(ctypes.byref(problem()), scorer, ctypes.byref(out)) == 0
        big = ctypes.c_size_t(0)
        assert lib.kvp_workspace_bytes(ctypes.byref(problem(S=4000, n_kept=500)), scorer, ctypes.byref(big)) == 0
        assert big.value > out.value > 0
        sizes.append(out.value)
    n = ctypes.c_int(0)
    assert lib.kvp_launches_per_compress(ctypes.byref(problem()), 99, ctypes.byref(n)) == -7


def test_header_is_valid_c_and_links_from_c(tmp_path):
    """include/kvpress_b200.h compiled as strict C99 by gcc, linked against the shared library, run without a GPU."""
    import shutil
    import subprocess

    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    native.load()
    lib = native.library_path()
    root = HEADER.parent.parent
    exe = tmp_path / "check_abi"
    subprocess.run([gcc, "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", f"-I{root / 'include'}",
                    str(root / "tests" / "c_abi" / "check_abi.c"), str(lib), f"-Wl,-rpath,{lib.parent}", "-o", str(exe)],
                   check=True, capture_output=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    assert out.startswith("abi 1 knorm_ws ")


def test_fused_knorm_queue_is_a_valid_schedule():
    """The item queue of the fused Knorm kernel (select_compact.cu: decode_fused_item) for both lags: every score /
    refine / compact item appears exactly once, and every item comes after the items it waits for (refine(row) after
    all score(row, .), compact(row, .) after all refine(row, .)) — the no-deadlock argument of the kernel."""
    import ctypes

    from kvpress_b200 import native

    lib = ctypes.CDLL(str(native.library_path()))
    fn = lib.kvp_debug_fused_queue_item
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_int] * 5 + [ctypes.c_longlong, ctypes.POINTER(ctypes.c_int)]
    out = (ctypes.c_int * 3)()
    for R, nT, lag, m_head in [(8, 10, 2, 0), (1, 3, 1, 1), (1, 3, 2, 0), (2, 7, 2, 0), (8, 64, 1, 32), (3, 5, 1, 0),
                               (5, 33, 1, 33), (4, 16, 1, 100), (2, 1, 1, 0), (9, 2, 2, 0)]:
        lag = min(lag, R)
        nA = (nT + 15) // 16
        total = R * (2 * nT + nA)
        seen, pos = set(), {}
        for item in range(total):
            assert fn(R, nT, nA, lag, m_head, item, out) == 0
            key = (out[0], out[1], out[2])
            assert key not in seen, (R, nT, lag, m_head, item, key)
            seen.add(key)
            pos[key] = item
        assert fn(R, nT, nA, lag, m_head, total, out) == -1
        want = {(0, r, i) for r in range(R) for i in range(nT)} | {(1, r, g) for r in range(R) for g in range(nA)} | \
               {(2, r, i) for r in range(R) for i in range(nT)}
        assert seen == want
        for r in range(R):
            last_score = max(pos[(0, r, i)] for i in range(nT))
            first_refine, last_refine = min(pos[(1, r, g)] for g in range(nA)), max(pos[(1, r, g)] for g in range(nA))
            first_compact = min(pos[(2, r, i)] for i in range(nT))
            assert last_score < first_refine and last_refine < first_compact
            if lag == 1 and r + 1 < R:  # the head of the next row's score items sits in front of the first compact item
                head = min(m_head, nT)
                assert all(pos[(0, r + 1, i)] < first_compact for i in range(head))


def test_ea_pair_kernel_partition_is_balanced_and_complete():
    """Work partition of the CTA-pair ExpectedAttention kernel (expected_attention.cu: ea2_start / ea2_pair_of): the
    (unit, tile-pair) items are cut into contiguous ranges, one per CTA pair. Every item belongs to exactly one pair,
    range sizes differ by at most one item, and for every unit the pairs that touch it are exactly
    [first, first + count) — the slots of the per-CTA softmax partials the kernel writes (two per pair) and the
    finalize kernel merges; slots beyond 2 * count are neutralised by the unit's first CTA."""
    import ctypes

    from kvpress_b200 import native

    lib = ctypes.CDLL(str(native.library_path()))
    fn = lib.kvp_debug_ea_pair_partition
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_int] * 5 + [ctypes.POINTER(ctypes.c_longlong)]
    out = (ctypes.c_longlong * 4)()
    for n_units, n_tp, n_pairs in [(16, 512, 74), (8, 512, 74), (1, 1024, 74), (4, 10, 40), (4, 10, 3), (3, 7, 21),
                                   (2, 1, 2), (1, 1, 1), (16, 512, 73), (5, 13, 64), (80, 512, 72)]:
        total = n_units * n_tp
        owner = [-1] * total
        sizes = []
        for p in range(n_pairs):
            assert fn(n_units, n_tp, n_pairs, p, 0, out) == 0
            lo, hi = out[0], out[1]
            assert 0 <= lo < hi <= total, (n_units, n_tp, n_pairs, p, lo, hi)   # n_pairs <= total: no empty range
            sizes.append(hi - lo)
            for i in range(lo, hi):
                assert owner[i] == -1
                owner[i] = p
        assert all(o >= 0 for o in owner) and max(sizes) - min(sizes) <= 1
        for u in range(n_units):
            assert fn(n_units, n_tp, n_pairs, 0, u, out) == 0
            first, count = out[2], out[3]
            touching = sorted(set(owner[u * n_tp:(u + 1) * n_tp]))
            assert touching == list(range(first, first + count)), (n_units, n_tp, n_pairs, u)
            assert 2 * count <= 160                                            # kEaMaxParts slots per (row, head)
    assert fn(4, 10, 41, 0, 0, out) == -1                                      # more pairs than items: the launcher clamps


def test_sources_read_no_environment_and_switch_on_no_kvp_macro():
    """What the library computes and which kernels it runs depend on its arguments alone: no source file calls getenv,
    and no preprocessor conditional names a KVP_ macro (a switch nothing defines leaves one side of it uncompiled and
    untested)."""
    csrc = HEADER.parent.parent / "kvpress_b200" / "csrc"
    files = sorted(f for f in csrc.rglob("*") if f.is_file())
    assert any(f.suffix == ".cu" for f in files)
    found = []
    for f in files:
        for n, line in enumerate(f.read_text().splitlines(), 1):
            if "getenv" in line or re.match(r"\s*#\s*(if|ifdef|ifndef|elif)\b.*\bKVP_", line):
                found.append(f"{f.name}:{n}: {line.strip()}")
    assert not found, found
