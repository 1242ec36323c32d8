"""The C ABI's status cases, shared by tests/test_abi_status_matrix.py and the per-press host tests.

An entry point has one valid call. Its cases are that call, each argument changed on its own (made invalid or set to
another valid value), and every pair of changes to two different arguments. The pointers are fake, 16-byte aligned or
not, and never dereferenced: the cases run in a child process that sees no GPU, so a call that passes every check
fails at its first CUDA call with KVP_ERR_CUDA (-6).

A press's entry points are checked against a restatement of the documented check order (include/kvpress_b200.h):
`expected` restates what every call shares (api.cu: validate -> n_kept == 0 short cut -> check_io -> the entry point's
operands -> the workspace), and the press's `Spec` states the rest.
"""
import ctypes
import importlib
import itertools
import json
import os
import subprocess
import sys
from dataclasses import dataclass, field
from pathlib import Path
from typing import Callable

ROOT = Path(__file__).resolve().parent.parent
GOOD, ODD16 = 0x10000, 0x1000C  # aligned; 4-byte but not 16-byte aligned
FIELDS = dict(B=1, Hkv=2, Hq=4, S=1000, D=128, n_kept=500, dtype=0)
STRIDES = (256000, 128000, 128)
PYTHON = [sys.executable, *(["-s"] if sys.flags.no_user_site else [])]


def child_env(**extra) -> dict:
    """This process's environment without the tests' KVP_* variables (KVP_RECORD_* re-records references), then
    `extra`."""
    env = {k: v for k, v in os.environ.items() if not k.startswith("KVP_")}
    env.update(extra)
    return env


def in_child(fn: str, *args):
    """What `fn(*args)` ("module:function") returns through JSON, run in a child process that sees no GPU."""
    module, name = fn.split(":")
    code = (f"import importlib, json; "
            f"print(json.dumps(getattr(importlib.import_module({module!r}), {name!r})(*{args!r})))")
    r = subprocess.run([*PYTHON, "-c", code], cwd=ROOT, env=child_env(CUDA_VISIBLE_DEVICES=""), capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def load_native():
    """kvpress_b200/native.py alone: importing the package would also import the presses and transformers, for
    nothing. Run only in a process that sees no GPU."""
    import importlib.util

    import torch

    assert torch.cuda.device_count() == 0, "the status cases pass fake device pointers: they must not see a GPU"
    spec = importlib.util.spec_from_file_location("kvp_native", ROOT / "kvpress_b200" / "native.py")
    nat = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(nat)
    return nat, nat.load()


def case_matrix(changes: dict) -> dict:
    """{case name: {slot: value}} from {slot: {label: changed value}}: the valid call, every single change and every
    pair of changes to two different slots, in that order."""
    singles = [(s, label, v) for s, c in changes.items() for label, v in c.items()]
    cases = {"valid": {}, **{f"{s}={label}": {s: v} for s, label, v in singles}}
    cases.update({f"{s1}={l1},{s2}={l2}": {s1: v1, s2: v2}
                  for (s1, l1, v1), (s2, l2, v2) in itertools.combinations(singles, 2) if s1 != s2})
    return cases


def problem(nat, changes: dict, fields: dict):
    """The kvp_problem of `fields` with the problem slots of `changes` applied."""
    p = nat.KvpProblem()
    for k, v in {**fields, **{k: v for k, v in changes.items() if k in FIELDS}}.items():
        setattr(p, k, v)
    p.k_stride = (ctypes.c_int64 * 3)(*changes.get("k_stride", STRIDES))
    p.v_stride = (ctypes.c_int64 * 3)(*changes.get("v_stride", STRIDES))
    return p


def workspace_bytes(lib, p, scorer: int) -> int:
    """What kvp_workspace_bytes asks for `p`; 1 MiB for a null or invalid problem, whose call fails before its
    workspace is looked at."""
    need = ctypes.c_size_t(1 << 20)
    if p is not None:
        lib.kvp_workspace_bytes(ctypes.byref(p), scorer, ctypes.byref(need))
    return need.value


def arg(slot: str, v, need: Callable[[], int]):
    """One argument as ctypes takes it. "enough" / "short" is the workspace `need()` asks for / one byte less."""
    if isinstance(v, str):
        if v == "sstride":
            return (ctypes.c_int64 * 2)(2000, 1000)
        return need() - (v == "short")
    if slot in ("idx", "inv_freq") and v is not None:
        return ctypes.cast(ctypes.c_void_p(v), ctypes.POINTER(ctypes.c_int32 if slot == "idx" else ctypes.c_float))
    return v


# --------------------------------------------------------------------------------------------------
# the entry points of one press
# --------------------------------------------------------------------------------------------------
@dataclass
class Spec:
    """What a press's score and compress entry points check beyond what every call checks.

    `operands` maps "score" / "compress" to (the operands that must not be null, those that must be 16-byte aligned),
    checked after check_io. `checks(f, a, compress)` are its argument checks in order: the first failing status, or 0.
    `short(f, a)` is the status of a workspace one byte short of what kvp_workspace_bytes asks for."""
    scorer: int
    slots: dict  # entry point -> its arguments after the kvp_problem
    valid: dict  # argument -> its valid value
    changes: dict  # slot -> {label: changed value}
    operands: dict
    checks: Callable[[dict, dict, bool], int]
    fields: dict = field(default_factory=dict)  # the press's valid problem, over FIELDS
    problem: tuple = ("dtype", "S", "D", "Hq", "n_kept", "v_stride")  # the problem slots changed
    short: Callable[[dict, dict], int] = lambda f, a: -5


def cases(spec: Spec, name: str) -> dict:
    return case_matrix({s: spec.changes.get(s, {}) for s in ["p", *spec.problem, *spec.slots[name].split()]})


def validate(c: dict, f: dict) -> int:
    """api.cu's validate()."""
    if c.get("p", 0) is None:
        return -1
    if f["dtype"] not in (0, 1):
        return -3
    if min(f["B"], f["Hkv"], f["S"], f["D"]) <= 0 or f["D"] % 8 or f["D"] > 256 or f["Hq"] <= 0 or f["Hq"] % f["Hkv"]:
        return -2
    if not 0 <= f["n_kept"] <= f["S"]:
        return -7
    if f["B"] * f["Hkv"] > 65535:
        return -2
    ks, vs = c.get("k_stride", STRIDES), c.get("v_stride", STRIDES)
    if any(x % 8 or x < 0 for x in ks + vs) or min(ks[2], vs[2]) < f["D"]:
        return -4
    return 0


def _pointers(nulls, aligned) -> int:
    if None in nulls:
        return -1
    return -4 if any(x % 16 for x in aligned) else 0


def expected(spec: Spec, name: str, c: dict) -> int:
    """The documented status of case `c` of entry point `name`: validate -> n_kept == 0 short cut (compress) ->
    K / V / outputs (compress) -> the operands of the call -> the press's argument checks -> workspace null ->
    alignment -> size."""
    f = {**FIELDS, **spec.fields, **{k: v for k, v in c.items() if k in FIELDS}}
    a = {**spec.valid, **{k: v for k, v in c.items() if k not in FIELDS}}
    compress = name.endswith("compress")
    rc = validate(c, f)
    if rc or (compress and f["n_kept"] == 0):
        return rc
    if compress:
        io = [a["K"], a["V"], a["K_out"], a["V_out"]]
        if rc := _pointers(io, io):
            return rc
    nulls, aligned = spec.operands["compress" if compress else "score"]
    rc = _pointers([a[x] for x in nulls], [a[x] for x in aligned]) or spec.checks(f, a, compress)
    if rc:
        return rc
    if a["ws"] is None:
        return -1
    if a["ws"] % 16:
        return -4
    return spec.short(f, a) if a["ws_bytes"] == "short" else -6


def statuses(module: str) -> dict:
    """The library's status of every case of the press whose test `module` holds its `ABI` spec. The workspace is
    sized for each case's problem. Run only in a process that sees no GPU."""
    spec = importlib.import_module(module).ABI
    nat, lib = load_native()
    fields = {**FIELDS, **spec.fields}
    out = {}
    for name in spec.slots:
        for label, c in cases(spec, name).items():
            pr = None if c.get("p", 0) is None else problem(nat, c, fields)
            args = [None if pr is None else ctypes.byref(pr)]
            for slot in spec.slots[name].split():
                args.append(arg(slot, c.get(slot, spec.valid[slot]), lambda: workspace_bytes(lib, pr, spec.scorer)))
            out[f"{name}({label})"] = getattr(lib, name)(*args)
    return out


def assert_statuses(module: str, floor: int) -> dict:
    """Every case of the press of `module` (more than `floor`) has its documented status. Returns the documented
    statuses by "entry point(case)"."""
    spec = importlib.import_module(module).ABI
    got = in_child("tests.abi_cases:statuses", module)
    want = {f"{name}({label})": expected(spec, name, c) for name in spec.slots for label, c in cases(spec, name).items()}
    assert sorted(got) == sorted(want) and len(got) > floor
    diffs = [f"{k}: {got[k]} != {want[k]}" for k in want if got[k] != want[k]]
    assert not diffs, f"{len(diffs)} differences, first ones:\n" + "\n".join(diffs[:30])
    return want
