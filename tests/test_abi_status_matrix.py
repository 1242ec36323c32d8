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
import itertools
import json
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
STORE = ROOT / "tests" / "golden" / "abi_status_matrix.json"
RECORD = os.environ.get("KVP_RECORD_ABI_STATUS") == "1"

GOOD, ODD, BIG = 0x10000, 0x1000C, 1 << 40  # aligned / misaligned pointer; more workspace than any case needs
FIELDS = dict(B=1, Hkv=2, Hq=4, S=1000, D=128, n_kept=500, dtype=0)
STRIDES = (256000, 128000, 128)
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


def _problem(native, changes=None, **fields):
    changes = changes or {}
    p = native.KvpProblem()
    for k, v in {**FIELDS, **fields, **{k: v for k, v in changes.items() if k in FIELDS}}.items():
        setattr(p, k, v)
    p.k_stride = (ctypes.c_int64 * 3)(*changes.get("k_stride", STRIDES))
    p.v_stride = (ctypes.c_int64 * 3)(*changes.get("v_stride", STRIDES))
    return p


def _call(native, lib, name, changes):
    """`name` with the valid arguments and `changes` ({slot: value}): its status, and for the two query calls the value
    written through the output pointer."""
    scorer, slots = ENTRIES[name]
    args, out = [None if changes.get("p", 0) is None else ctypes.byref(_problem(native, changes))], None
    for slot in slots.split():
        v = changes.get(slot, ARGS[slot][0] if slot in ARGS else GOOD)
        if v == "out":
            out = (ctypes.c_size_t if name == "kvp_workspace_bytes" else ctypes.c_int)(0)
            v = ctypes.byref(out)
        elif v == "sstride":
            v = (ctypes.c_int64 * 2)(2000, 1000)
        elif v == "short":  # one byte less than the library asks for the valid problem
            need = ctypes.c_size_t(0)
            assert lib.kvp_workspace_bytes(ctypes.byref(_problem(native)), scorer, ctypes.byref(need)) == 0
            v = need.value - 1
        elif slot in ("idx", "inv_freq") and v is not None:
            v = ctypes.cast(ctypes.c_void_p(v), ctypes.POINTER(ctypes.c_int32 if slot == "idx" else ctypes.c_float))
        args.append(v)
    rc = getattr(lib, name)(*args)
    return str(-rc) if out is None else f"{-rc}:{out.value}"


def matrix() -> dict:
    """Every case, per entry point: a digest of the case names and the results in case order. Run only in a process
    that sees no GPU."""
    import importlib.util

    import torch

    assert torch.cuda.device_count() == 0, "the status matrix passes fake device pointers: it must not see a GPU"
    # the binding alone: importing the package would also import the presses and transformers, for nothing
    spec = importlib.util.spec_from_file_location("kvp_native", ROOT / "kvpress_b200" / "native.py")
    native = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(native)
    lib = native.load()
    got = {}
    for name, (_, slots) in ENTRIES.items():
        changes = {**PROBLEM_CHANGES, **{s: ARGS[s][1] if s in ARGS else PTR for s in slots.split()}}
        singles = [(s, label, v) for s, c in changes.items() for label, v in c.items()]
        cases = {"valid": {}, **{f"{s}={label}": {s: v} for s, label, v in singles}}
        cases.update({f"{s1}={l1},{s2}={l2}": {s1: v1, s2: v2}
                      for (s1, l1, v1), (s2, l2, v2) in itertools.combinations(singles, 2) if s1 != s2})
        results = [_call(native, lib, name, c) for c in cases.values()]
        got[name] = {"cases": hashlib.sha256("|".join(cases).encode()).hexdigest()[:16], "names": list(cases),
                     "results": "".join(results) if all(len(r) == 1 for r in results) else " ".join(results)}
    for B, H, G, S, D in SWEEP:
        p = ctypes.byref(_problem(native, B=B, Hkv=H, Hq=G * H, S=S, D=D, n_kept=S // 2))
        row = []
        for scorer in range(6):
            n, launches = ctypes.c_size_t(0), ctypes.c_int(0)
            assert lib.kvp_workspace_bytes(p, scorer, ctypes.byref(n)) == 0
            assert lib.kvp_launches_per_compress(p, scorer, ctypes.byref(launches)) == 0
            row.append([n.value, launches.value])
        got.setdefault(f"sizes B{B} Hkv{H} G{G}", {})[f"S{S} D{D}"] = row
    return got


def test_every_status_workspace_size_and_launch_count_matches_the_recording():
    env = {k: v for k, v in os.environ.items() if not k.startswith("KVP_")}  # the library's knobs at their defaults
    env["CUDA_VISIBLE_DEVICES"] = ""
    code = "import json, tests.test_abi_status_matrix as m; print(json.dumps(m.matrix()))"
    r = subprocess.run([sys.executable, *(["-s"] if sys.flags.no_user_site else []), "-c", code], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
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
