"""Host behaviour of the C ABI, pinned exactly against tests/golden/abi_status_matrix.json: the status of every entry
point that takes a kvp_problem, and what kvp_workspace_bytes / kvp_launches_per_compress answer.

Each entry point has one valid call. The cases are that call, each argument changed on its own (made invalid or set
to another valid value), and every pair of changes to two different arguments. The pairs pin which check wins when two
arguments are bad, including n_kept = 0 with each bad operand. The workspace is also given one byte less than
kvp_workspace_bytes. The two query calls are also swept over shapes for all six scorer ids, on both sides of the Knorm
cluster / fused / two-kernel boundaries.

The pointers are fake, 16-byte aligned or not, and never dereferenced: the matrix runs in a child process that sees
no GPU. A call that passes every check fails at its first CUDA call with KVP_ERR_CUDA, so a recorded -6 means "passes
validation". To re-record from the library as built:  KVP_RECORD_ABI_STATUS=1 python -m pytest <this file>
"""
import ctypes
import hashlib
import json
import os
from pathlib import Path

from tests.abi_cases import FIELDS, GOOD, ODD16 as ODD, arg, case_matrix, in_child, load_native, problem, \
    workspace_bytes

STORE = Path(__file__).resolve().parent / "golden" / "abi_status_matrix.json"
RECORD = os.environ.get("KVP_RECORD_ABI_STATUS") == "1"

BIG = 1 << 40  # more workspace than any case needs
BAD_STRIDES = {"s100": (256000, 128000, 100), "s120": (256000, 128000, 120), "b-8": (-8, 128000, 128)}
PROBLEM_CHANGES = {  # slot -> {label: value}
    "p": {"null": None},
    "B": {"0": 0, "40000": 40000},  # 40000 * Hkv rows exceed gridDim.y
    "Hkv": {"0": 0, "3": 3},
    "Hq": {"0": 0, "5": 5, "8": 8},
    "S": {"0": 0, "499": 499, "4000": 4000},
    "D": {"0": 0, "12": 12, "24": 24, "264": 264},  # 24: valid except for the re-rotating compaction
    "n_kept": {"0": 0, "-1": -1, "1000": 1000, "1001": 1001},
    "dtype": {"f16": 1, "3": 3},
    "k_stride": BAD_STRIDES,
    "v_stride": BAD_STRIDES,
}
PTR = {"null": None, "odd": ODD}
# argument after the problem -> (valid value, {label: changed value})
ARGS = {
    "scorer": (1, {str(i): i for i in (0, 2, 3, 4, 5, 99, -1)}),
    "out": ("out", {"null": None}),
    "ws": (GOOD, PTR),
    "ws_bytes": (BIG, {"short": "short", "64": 64}),
    "sstride": ("sstride", {"null": None}),
    "n_sink": (4, {"-1": -1, "0": 0, "999": 999, "1000": 1000}),
    "window": (64, {"0": 0, "256": 256, "999": 999, "1000": 1000}),
    "kernel_size": (5, {"0": 0, "4": 4, "1": 1, "-1": -1}),
    "epsilon": (0.25, {}),
    "use_vnorm": (1, {"0": 0}),
    "stream": (0, {}),
}
IO, WS = "K V K_out V_out idx", "ws ws_bytes stream"
ENTRIES = {  # entry point -> (scorer whose workspace it takes, its arguments after the problem)
    "kvp_workspace_bytes": (None, "scorer out"),
    "kvp_launches_per_compress": (None, "scorer out"),
    "kvp_workspace_check": (1, f"scorer {WS}"),
    "kvp_knorm_score": (None, "K scores stream"),
    "kvp_knorm_compress": (1, f"{IO} scores {WS}"),
    "kvp_keydiff_score": (5, f"K scores {WS}"),
    "kvp_keydiff_compress": (5, f"{IO} scores {WS}"),
    "kvp_streaming_score": (None, "n_sink scores stream"),
    "kvp_streaming_compress": (None, f"n_sink {IO} stream"),
    "kvp_snapkv_score": (3, f"K q window kernel_size scores {WS}"),
    "kvp_snapkv_compress": (3, f"K V q window kernel_size K_out V_out idx scores {WS}"),
    "kvp_expected_attention_score": (4, f"K V mu cov epsilon n_sink use_vnorm scores {WS}"),
    "kvp_expected_attention_compress": (4, f"K V mu cov epsilon n_sink use_vnorm K_out V_out idx scores {WS}"),
    "kvp_scores_compress": (0, f"scores sstride {IO} {WS}"),
    "kvp_scores_select": (0, f"scores sstride idx {WS}"),
    "kvp_scores_compress_rerotate": (0, f"scores sstride K V inv_freq K_out V_out idx {WS}"),
}
# (B, Hkv, Hq / Hkv, S, D): the sweep, the Knorm cluster kernel's limits, and 32 MiB of K beyond its reach
SWEEP = [(2, 4, G, S, D) for G in (1, 3, 4, 8) for S in (1, 255, 256, 257, 2560, 131072) for D in (8, 64, 96, 128, 256)]
SWEEP += [(1, 8, 1, S, D) for D in (64, 128, 256) for S in (3072, 3073, 3080, 3081, 5888, 5889, 5896, 5897, 6144, 6145)]
SWEEP += [(1, 1, 1, 131072, 128), (1, 1, 1, 131073, 128), (2, 8, 1, 8192, 128), (2, 8, 1, 8193, 128),
          (2, 1, 1, 131072, 64), (2, 1, 1, 131073, 64)]


def _call(native, lib, name, changes):
    """`name` with the valid arguments and `changes` ({slot: value}): its status, and for the two query calls the value
    written through the output pointer."""
    scorer, slots = ENTRIES[name]
    args, out = [None if changes.get("p", 0) is None else ctypes.byref(problem(native, changes, FIELDS))], None
    for slot in slots.split():
        v = changes.get(slot, ARGS[slot][0] if slot in ARGS else GOOD)
        if v == "out":
            out = (ctypes.c_size_t if name == "kvp_workspace_bytes" else ctypes.c_int)(0)
            v = ctypes.byref(out)
        else:  # "short": one byte less than the library asks for the valid problem
            v = arg(slot, v, lambda: workspace_bytes(lib, problem(native, {}, FIELDS), scorer))
        args.append(v)
    rc = getattr(lib, name)(*args)
    return str(-rc) if out is None else f"{-rc}:{out.value}"


def matrix() -> dict:
    """Every case, per entry point: a digest of the case names and the results in case order. Run only in a process
    that sees no GPU."""
    native, lib = load_native()
    got = {}
    for name, (_, slots) in ENTRIES.items():
        cases = case_matrix({**PROBLEM_CHANGES, **{s: ARGS[s][1] if s in ARGS else PTR for s in slots.split()}})
        results = [_call(native, lib, name, c) for c in cases.values()]
        got[name] = {"cases": hashlib.sha256("|".join(cases).encode()).hexdigest()[:16], "names": list(cases),
                     "results": "".join(results) if all(len(r) == 1 for r in results) else " ".join(results)}
    for B, H, G, S, D in SWEEP:
        p = ctypes.byref(problem(native, {}, dict(FIELDS, B=B, Hkv=H, Hq=G * H, S=S, D=D, n_kept=S // 2)))
        row = []
        for scorer in range(6):
            n, launches = ctypes.c_size_t(0), ctypes.c_int(0)
            assert lib.kvp_workspace_bytes(p, scorer, ctypes.byref(n)) == 0
            assert lib.kvp_launches_per_compress(p, scorer, ctypes.byref(launches)) == 0
            row.append([n.value, launches.value])
        got.setdefault(f"sizes B{B} Hkv{H} G{G}", {})[f"S{S} D{D}"] = row
    return got


def test_every_status_workspace_size_and_launch_count_matches_the_recording():
    got = in_child(f"{__name__}:matrix")
    names = {k: v.pop("names") for k, v in got.items() if "names" in v}
    if RECORD:
        STORE.write_text("{\n" + ",\n".join(f"{json.dumps(k)}: {json.dumps(v)}" for k, v in got.items()) + "\n}\n")
    want = json.loads(STORE.read_text())
    assert sorted(got) == sorted(want)
    diffs = []
    for key, w in want.items():
        g = got[key]
        if key in names:
            assert g["cases"] == w["cases"], f"{key}: the cases changed; re-record the matrix"
            split = (lambda s: s.split(" ")) if " " in w["results"] else list
            diffs += [f"{key}({case}): {a} != {b} (negated status)"
                      for case, a, b in zip(names[key], split(g["results"]), split(w["results"])) if a != b]
        else:
            diffs += [f"{key} {shape}: [workspace bytes, launches] per scorer {g.get(shape)} != {row}"
                      for shape, row in w.items() if g.get(shape) != row]
            assert sorted(g) == sorted(w), key
    assert not diffs, f"{len(diffs)} differences, first ones:\n" + "\n".join(diffs[:30])
    assert sum(len(n) for n in names.values()) > 10000
