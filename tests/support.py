"""Helpers shared by the host tests: the record / replay store of the unmodified reference's results, the signatures
and tolerance its results are compared with, and a recording stand-in for the shared library."""
import contextlib
import ctypes
import os
import sys
import types

import numpy as np
import pytest
import torch

from kvpress_b200 import native
from tests.conftest import GOLDEN_DIR

# down-casts applied to the reference's results before they are stored
TO_INT32 = {np.dtype(np.int64): np.int32}
TO_32BIT = {np.dtype(np.float64): np.float32, **TO_INT32}  # float32 is well inside the comparison tolerance


def import_reference():
    from oracle.build_ref import REFERENCE

    path = str(REFERENCE)
    assert (REFERENCE / "kvpress").is_dir(), "recording needs a reference checkout (oracle/build_ref.py)"
    sys.modules.setdefault("fire", types.ModuleType("fire"))
    if path not in sys.path:
        sys.path.insert(0, path)
    import kvpress

    return kvpress


def reference_store(store, record_env: str, casts: dict = None, merge: bool = False):
    """A module-scoped fixture `ref(key, compute)`. With `record_env`=1 it runs `compute(kvpress)` on the unmodified
    reference, stores the results (each array down-cast by `casts`) in the .npz `store` when the module is done and
    returns them; with `merge` the new results are added to the stored ones instead of replacing them. Otherwise it
    returns the stored results of `key`."""
    record = os.environ.get(record_env) == "1"
    casts = casts or {}

    @pytest.fixture(scope="module")
    def ref():
        stored = {} if record or not store.exists() else dict(np.load(store))
        recorded = {}

        def result(key: str, compute) -> dict:
            if record:
                out = {k: np.asarray(x.detach().numpy() if torch.is_tensor(x) else x)
                       for k, x in compute(import_reference()).items()}
                out = {k: x.astype(casts[x.dtype]) if x.dtype in casts else x for k, x in out.items()}
                recorded.update({f"{key}|{k}": x for k, x in out.items()})
                return out
            out = {k.split("|", 1)[1]: x for k, x in stored.items() if k.split("|", 1)[0] == key}
            assert out, f"no stored reference result for {key}"
            return out

        yield result
        if record:
            old = dict(np.load(store)) if merge and store.exists() else {}
            np.savez_compressed(store, **{**old, **recorded})

    return ref


def close(got, want, what=""):
    """Same values up to float32 rounding of another host: the stored values come from another host's float32 CPU
    kernels, and a different retained row differs by orders of magnitude more."""
    got, want = (torch.as_tensor(x.detach() if torch.is_tensor(x) else np.asarray(x), dtype=torch.float64)
                 for x in (got, want))
    assert got.shape == want.shape, (what, got.shape, want.shape)
    assert torch.allclose(got, want, rtol=1e-5, atol=1e-6), (what, float((got - want).abs().max()))


def ordered_signature(keys, values):
    """Signature of every retained (K, V) row of every head, in cache order: a seeded random projection."""
    g = torch.Generator().manual_seed(0)
    w = torch.randn(keys.shape[-1], generator=g, dtype=torch.float64)
    return keys.double() @ w + 3.0 * (values.double() @ w)


def rows_signature(keys, values):
    """Order-independent signature of the retained (K, V) rows of every head."""
    return ordered_signature(keys, values).sort(-1).values


# --------------------------------------------------------------------------------------------------
# a recording stand-in for the shared library
# --------------------------------------------------------------------------------------------------
class Recorder:
    def __init__(self, real):
        self.real, self.calls = real, []

    def __getattr__(self, name):
        if name in ("kvp_workspace_bytes", "kvp_launches_per_compress", "kvp_status_string", "kvp_last_cuda_error",
                    "kvp_abi_version"):
            return getattr(self.real, name)

        def fn(*args):
            p = args[0]._obj
            snap = {f: getattr(p, f) for f in ("B", "Hkv", "Hq", "S", "D", "n_kept", "dtype")}
            snap["k_stride"], snap["v_stride"] = tuple(p.k_stride), tuple(p.v_stride)
            vals = []
            for a in args[1:]:
                if isinstance(a, ctypes.c_void_p):
                    vals.append(a.value or 0)
                elif isinstance(a, ctypes.Array):
                    vals.append(tuple(a))
                else:
                    vals.append(a)
            self.calls.append((name, snap, vals))
            return 0
        return fn


@pytest.fixture
def rec(monkeypatch):
    """native's wrappers on CPU tensors, each call recorded as (entry point, kvp_problem fields, the other arguments)
    instead of run; the real library still answers kvp_workspace_bytes / kvp_launches_per_compress."""
    r = Recorder(native.load())
    monkeypatch.setattr(native, "load", lambda: r)
    monkeypatch.setattr(native, "_require_cuda_kv", lambda *a, **k: None)
    monkeypatch.setattr(native, "_stream", lambda: ctypes.c_void_p(0))
    monkeypatch.setattr(native, "_out_device", lambda keys: keys.device)
    monkeypatch.setattr(native, "_normalise", lambda t: t if native._rows_ok(t) else t.contiguous())  # CPU stands in for CUDA
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    # the recorder accepts any shape: keep the tiny head_dim-16 inputs of these tests on the C-ABI entry points
    from kvpress_b200 import wide_head_scores

    monkeypatch.setattr(wide_head_scores, "snapkv_on_tensor_cores", lambda *a: True)
    monkeypatch.setattr(wide_head_scores, "expected_attention_on_tensor_cores", lambda *a: True)
    return r


def kv(B=2, H=3, S=50, D=64, dtype=torch.bfloat16):
    return torch.randn(B, H, S, D).to(dtype), torch.randn(B, H, S, D).to(dtype)


def rerotation_cases():
    """Per case: the regenerated inputs (checked against the stored checksum) and a getter of the stored arrays; the
    reference's re-rotated outputs are stored as SHA-256 digests (make_golden.digest16)."""
    from tests.golden.make_golden import RERO_CASES, rerotation_inputs, tensor_checksum

    z = np.load(GOLDEN_DIR / "rerotation.npz")
    for (tag, B, H, S, D, dtype, theta), row in zip(RERO_CASES, z["cases"]):
        assert row.tolist() == [B, H, S, D, int(dtype == torch.float16)]
        inputs = rerotation_inputs(B, H, S, D, dtype, theta)
        assert (tensor_checksum(*inputs[:2], inputs[3]) == z[f"{tag}_checksum"]).all(), "RNG no longer reproduces"
        get = lambda k, tag=tag: z[f"{tag}_{k}"]  # noqa: E731
        yield tag, int(S), [float(r) for r in z["ratios"]], inputs, get
