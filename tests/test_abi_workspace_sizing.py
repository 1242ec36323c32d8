"""kvp_workspace_bytes sizes the workspace of every call its scorer's entry points accept, whatever the call's other
arguments: a call given exactly the bytes it asks for never returns KVP_ERR_WORKSPACE_TOO_SMALL.

Per scorer, over a grid of problems and of the arguments each entry point accepts (SnapKV: every group size 1 ... 8 and
the windows at the edges of 1 ... 512 / G; ObservedAttention: n_q from 1 to S; CUR: r from 0 to 32 with local windows
0, 1 and 1024; ...), the valid call on exactly that many bytes passes every check. The pointers are fake, 16-byte
aligned and never dereferenced: the calls run in a child process that sees no GPU, so a call that passes every check
fails at its first CUDA call with KVP_ERR_CUDA (-6). SnapKV's size is also pinned from above: its largest window on
one byte less is too small.
"""
import ctypes

from tests.abi_cases import GOOD, in_child, load_native

OK_CUDA, TOO_SMALL = -6, -5
SNAP_MAX_ROWS = 512  # kSnapMaxRows: G * window query rows per kv head


def _problem(nat, B, Hkv, G, S, D, n_kept, dtype=0):
    p = nat.KvpProblem()
    p.B, p.Hkv, p.Hq, p.S, p.D, p.n_kept, p.dtype = B, Hkv, Hkv * G, S, D, n_kept, dtype
    p.k_stride = (ctypes.c_int64 * 3)(Hkv * S * D, S * D, D)
    p.v_stride = (ctypes.c_int64 * 3)(Hkv * S * D, S * D, D)
    return p


def _kept(S: int) -> list:
    """n_kept = 1, an odd middle value, S - 1 and S"""
    return sorted({1, (S // 2) | 1 if S > 2 else 1, max(1, S - 1), S})


def _snap_windows(G: int, S: int) -> list:
    top = min(SNAP_MAX_ROWS // G, S - 1)
    edges = {1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257, 300, 384, 511, top - 1, top}
    return sorted(w for w in edges if 1 <= w <= top)


def calls():
    """[(label, status, short)]: every call on exactly kvp_workspace_bytes bytes, and for SnapKV's largest window the
    status of the same call on one byte less (else None). Run only in a process that sees no GPU."""
    nat, lib = load_native()
    out = []
    sstride_of = lambda Hkv, S: (ctypes.c_int64 * 2)(Hkv * S, S)  # noqa: E731

    def run(label, scorer, name, shape, n_kept, args, short=False):
        p = _problem(nat, *shape, n_kept)
        need = ctypes.c_size_t(0)
        assert lib.kvp_workspace_bytes(ctypes.byref(p), scorer, ctypes.byref(need)) == 0, label
        fn = getattr(lib, name)
        rc = fn(ctypes.byref(p), *args, GOOD, need.value, None)
        tight = fn(ctypes.byref(p), *args, GOOD, need.value - 1, None) if short else None
        out.append((f"{name}{shape} n_kept={n_kept} {label}", rc, tight))

    io = (GOOD,) * 5  # K, V, K_out, V_out, idx
    tc_shapes = [(B, Hkv, G, S, D) for D in (64, 128) for (B, Hkv, G, S) in (
        (1, 1, 1, 2), (3, 1, 1, 257), (1, 5, 2, 1000), (1, 32, 1, 4096), (1, 8, 4, 32768), (2, 2, 8, 4097),
        (1, 4, 3, 512), (1, 2, 7, 131072))]

    # SnapKV: every G in 1 ... 8, the windows at the edges of [1, min(512 / G, S - 1)]
    for D in (64, 128):
        for G in range(1, 9):
            for B, Hkv, S in ((1, 1, 2), (3, 1, 257), (1, 8, 1000), (1, 32, 4096), (1, 8, 32768), (1, 2, 131072)):
                for w in _snap_windows(G, S):
                    largest = w == min(SNAP_MAX_ROWS // G, S - 1)
                    run(f"w={w}", 3, "kvp_snapkv_score", (B, Hkv, G, S, D), 0, (GOOD, GOOD, w, 5, GOOD), largest)
                    run(f"w={w}", 3, "kvp_snapkv_compress", (B, Hkv, G, S, D), S // 2 or 1,
                        (GOOD, GOOD, GOOD, w, 5, GOOD, GOOD, GOOD, GOOD), largest)

    for shape in tc_shapes:
        B, Hkv, G, S, D = shape
        for n in _kept(S):
            # ExpectedAttention: with and without covariance / value norms, every n_sink
            for cov in (GOOD, None):
                for vn in (0, 1):
                    for n_sink in sorted({0, 4 % S, S - 1}):
                        a = (GOOD, GOOD, GOOD, cov, 0.0, n_sink, vn)
                        run(f"cov={bool(cov)} vnorm={vn} sink={n_sink}", 4, "kvp_expected_attention_compress", shape,
                            n, (*a, GOOD, GOOD, GOOD, GOOD))
                        if n == S:
                            run(f"cov={bool(cov)} vnorm={vn} sink={n_sink}", 4, "kvp_expected_attention_score", shape,
                                0, (*a, GOOD))
            # ObservedAttention: n_q from 1 to S
            for n_q in sorted({1, min(2, S), min(64, S), S // 2 or 1, S - 1 or 1, S}):
                if n == S:
                    run(f"n_q={n_q}", 7, "kvp_observed_attention_score", shape, 0, (GOOD, GOOD, n_q, 0.125, GOOD))
                run(f"n_q={n_q}", 7, "kvp_observed_attention_compress", shape, n,
                    (GOOD, GOOD, GOOD, n_q, 0.125, GOOD, GOOD, GOOD, GOOD))
            # CriticalKV: n_first 0 and n_kept (compress), 0 and S (score)
            sst, wo = sstride_of(Hkv, S), (4096, Hkv * G * D)
            for n_first in (0, n):
                run(f"n_first={n_first}", 6, "kvp_criticalkv_compress", shape, n,
                    (GOOD, GOOD, GOOD, sst, GOOD, *wo, 1e-4, n_first, GOOD, GOOD, GOOD, GOOD))
            if n == S:
                for n_first in (0, S):
                    run(f"n_first={n_first}", 6, "kvp_criticalkv_score", shape, 0,
                        (GOOD, GOOD, sst, GOOD, *wo, 1e-4, n_first, GOOD))
            # NonCausalAttention: chunk sizes 128 and 256
            for cs in (128, 256):
                if n == S:
                    run(f"cs={cs}", 8, "kvp_non_causal_attention_score", shape, 0, (GOOD, GOOD, GOOD, cs, GOOD))
                run(f"cs={cs}", 8, "kvp_non_causal_attention_compress", shape, n,
                    (GOOD, GOOD, GOOD, cs, GOOD, GOOD, GOOD, GOOD))

    # every head_dim: CUR, LagKV, KeyDiff, Knorm, Merging and the generic selection
    any_d = [(B, Hkv, G, S, D) for D in (8, 72, 128, 256) for (B, Hkv, G, S) in (
        (1, 1, 1, 1), (3, 1, 1, 257), (1, 5, 2, 1000), (2, 8, 4, 4097), (1, 2, 1, 65536))]
    for shape in any_d:
        B, Hkv, G, S, D = shape
        sst = sstride_of(Hkv, S)
        for n in _kept(S):
            first = n == _kept(S)[0]
            # CUR: r from 0 to 32, local windows 0, 1 and 1024, every leverage type
            for r in (0, 1, 7, 16, 31, 32) if first else (0, 32):
                for w in (0, 1, 1024):
                    for lt in range(4) if first else (3,):
                        g = GOOD if r else None
                        run(f"r={r} w={w} type={lt}", 11, "kvp_cur_compress", shape, n,
                            (GOOD, GOOD, 4, lt, w, g, r, GOOD, GOOD, GOOD, GOOD))
                        if first:
                            run(f"r={r} w={w} type={lt}", 11, "kvp_cur_score", shape, 0,
                                (GOOD, GOOD, 4, lt, w, g, r, GOOD))
            # LagKV: lag sizes 1 and 1024, cross scoring on and off
            for lag in (1, 1024):
                for cross in (0, 1):
                    run(f"lag={lag} cross={cross}", 9, "kvp_lagkv_compress", shape, n,
                        (GOOD, GOOD, 4, lag, cross, GOOD, GOOD, GOOD, GOOD))
                    if first:
                        run(f"lag={lag} cross={cross}", 9, "kvp_lagkv_score", shape, 0,
                            (GOOD, GOOD, 4, lag, cross, GOOD))
            if first:
                run("", 5, "kvp_keydiff_score", shape, 0, (GOOD, GOOD))
            run("", 5, "kvp_keydiff_compress", shape, n, (*io, GOOD))
            run("", 1, "kvp_knorm_compress", shape, n, (*io, GOOD))
            # Merging: both entry points
            for frac in (0.5, 1.0):
                run(f"frac={frac}", 13, "kvp_merging_compress", shape, n,
                    (GOOD, sst, GOOD, GOOD, 0.0, frac, GOOD, GOOD, GOOD, GOOD, GOOD))
                run(f"frac={frac}", 13, "kvp_merging_merge", shape, n,
                    (GOOD, GOOD, GOOD, 0.0, frac, GOOD, GOOD, GOOD))
            # generic selection
            run("", 0, "kvp_scores_select", shape, n, (GOOD, sst, GOOD))
            run("", 0, "kvp_scores_compress", shape, n, (GOOD, sst, *io))
            if D % 16 == 0:
                run("", 0, "kvp_scores_compress_rerotate", shape, n, (GOOD, sst, GOOD, GOOD, GOOD, GOOD, GOOD, GOOD))

    # Knorm: both sides of the cluster kernel's limits and of the fused kernel's 32 MiB of K
    for D in (64, 128, 256):
        for S in (3072, 3073, 3080, 3081, 5888, 5889, 5896, 5897, 6144, 6145):
            run("", 1, "kvp_knorm_compress", (1, 8, 1, S, D), S // 2, (*io, GOOD))
    for shape in ((1, 1, 1, 131072, 128), (1, 1, 1, 131073, 128), (2, 8, 1, 8192, 128), (2, 8, 1, 8193, 128),
                  (2, 1, 1, 131072, 64), (2, 1, 1, 131073, 64)):
        run("", 1, "kvp_knorm_compress", shape, shape[3] // 2, (*io, GOOD))
    launches = set()
    for D in (64, 128):
        for S in (3072, 6145, 131072, 131073):
            n = ctypes.c_int(0)
            lib.kvp_launches_per_compress(ctypes.byref(_problem(nat, 1, 8 if S < 10000 else 1, 1, S, D, S // 2)), 1,
                                          ctypes.byref(n))
            launches.add(n.value)
    out.append(("knorm paths", sorted(launches), None))
    return out


def test_every_accepted_call_fits_in_the_workspace_it_asks_for():
    got = in_child(f"{__name__}:calls")
    *got, (_, knorm_paths, _) = got
    assert knorm_paths == [1, 2, 3], "the Knorm grid no longer reaches the cluster, fused and two-kernel paths"
    bad = [f"{label}: {rc}" for label, rc, _ in got if rc != OK_CUDA]
    assert not bad, f"{len(bad)} of {len(got)} calls did not reach CUDA on exactly their workspace, first ones:\n" + \
        "\n".join(bad[:30])
    loose = [label for label, _, tight in got if tight is not None and tight != TOO_SMALL]
    assert not loose, f"SnapKV's largest window fits in one byte less than asked for:\n" + "\n".join(loose[:30])
    names = {label.split("(")[0] for label, _, _ in got}
    assert len(names) == 22, sorted(names)
    assert len(got) > 5000 and sum(tight is not None for *_, tight in got) > 50
