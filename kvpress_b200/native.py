"""ctypes binding of libkvpress_b200.so (the C ABI in include/kvpress_b200.h).

torch is used here only as the owner of device memory and streams: tensors are handed to the
library as raw pointers + element strides, outputs and scratch are allocated with torch's caching
allocator, kernels are enqueued on torch's current stream. There is NO fallback: if the shared
library is missing or a tensor is not a CUDA tensor, calls raise.
"""
from __future__ import annotations

import contextlib
import ctypes
import os
from pathlib import Path
from typing import Optional

import torch

_LIB_NAME = "libkvpress_b200.so"
_LIB_PATH = Path(__file__).resolve().parent / _LIB_NAME

(SCORER_GENERIC, SCORER_KNORM, SCORER_STREAMING, SCORER_SNAPKV, SCORER_EXPECTED_ATTENTION, SCORER_KEYDIFF,
 SCORER_CRITICALKV, SCORER_OBSERVED_ATTENTION, SCORER_NON_CAUSAL_ATTENTION, SCORER_LAGKV) = range(10)
SCORER_CUR = 11  # KVP_SCORER_CUR; id 10 is not assigned
SCORER_MERGING = 13  # KVP_SCORER_MERGING; id 12 is not assigned
SCORER_THINK = 14  # KVP_SCORER_THINK: kvp_think_prune
SCORER_FINCH = 16  # KVP_SCORER_FINCH: kvp_finch_*, kvp_scores_compress_chunked; id 15 is not assigned
SCORER_CAM = 17  # KVP_SCORER_CAM: kvp_cam_compress
SCORER_KVZAP = 18  # KVP_SCORER_KVZAP: kvp_kvzap_*
KVZAP_MAX_HIDDEN = 16384  # the shapes the KVzap kernels take (kZapMax* in csrc/common.cuh)
KVZAP_MAX_HD = 2048
KVZAP_MAX_HEADS = 32
LAG_MAX = 1024  # the largest lag_size the LagKV kernel scores (kLagMax in csrc/common.cuh)
CUR_WINDOW_MAX = 1024  # the largest local_window_size the CUR kernel scores (kCurWindowMax in csrc/common.cuh)
CUR_RANK_MAX = 32  # the most projection columns the CUR kernel scores (kCurRankMax)
CUR_LEVERAGE_TYPES = ("key", "value", "kv_avg", "kv_product")  # leverage_type 0 ... 3 of kvp_cur_score
_DTYPES = {torch.bfloat16: 0, torch.float16: 1}


class KvpProblem(ctypes.Structure):
    """Mirror of `struct kvp_problem`."""

    _fields_ = [
        ("B", ctypes.c_int32),
        ("Hkv", ctypes.c_int32),
        ("Hq", ctypes.c_int32),
        ("S", ctypes.c_int32),
        ("D", ctypes.c_int32),
        ("n_kept", ctypes.c_int32),
        ("dtype", ctypes.c_int32),
        ("reserved", ctypes.c_int32),
        ("k_stride", ctypes.c_int64 * 3),
        ("v_stride", ctypes.c_int64 * 3),
    ]


class NativeLibraryError(RuntimeError):
    pass


# name -> (restype, argtypes); every symbol include/kvpress_b200.h declares
_P = ctypes.c_void_p
_PP = ctypes.POINTER(KvpProblem)
_SZ = ctypes.c_size_t
_I = ctypes.c_int32
_I64 = ctypes.c_int64
_PI64 = ctypes.POINTER(ctypes.c_int64)
SIGNATURES = {
    "kvp_abi_version": (ctypes.c_int, []),
    "kvp_status_string": (ctypes.c_char_p, [ctypes.c_int]),
    "kvp_last_cuda_error": (ctypes.c_char_p, []),
    "kvp_workspace_bytes": (ctypes.c_int, [_PP, ctypes.c_int, ctypes.POINTER(_SZ)]),
    "kvp_launches_per_compress": (ctypes.c_int, [_PP, ctypes.c_int, ctypes.POINTER(ctypes.c_int)]),
    "kvp_workspace_check": (ctypes.c_int, [_PP, ctypes.c_int, _P, _SZ, _P]),
    "kvp_knorm_score": (ctypes.c_int, [_PP, _P, _P, _P]),
    "kvp_knorm_compress": (ctypes.c_int, [_PP, _P, _P, _P, _P, _P, _P, _P, _SZ, _P]),
    "kvp_streaming_score": (ctypes.c_int, [_PP, _I, _P, _P]),
    "kvp_streaming_compress": (ctypes.c_int, [_PP, _I, _P, _P, _P, _P, _P, _P]),
    "kvp_snapkv_score": (ctypes.c_int, [_PP, _P, _P, _I, _I, _P, _P, _SZ, _P]),
    "kvp_snapkv_compress": (ctypes.c_int, [_PP, _P, _P, _P, _I, _I, _P, _P, _P, _P, _P, _SZ, _P]),
    "kvp_expected_attention_score": (
        ctypes.c_int, [_PP, _P, _P, _P, _P, ctypes.c_float, _I, _I, _P, _P, _SZ, _P]),
    "kvp_expected_attention_compress": (
        ctypes.c_int, [_PP, _P, _P, _P, _P, ctypes.c_float, _I, _I, _P, _P, _P, _P, _P, _SZ, _P]),
    "kvp_scores_compress": (
        ctypes.c_int, [_PP, _P, ctypes.POINTER(ctypes.c_int64), _P, _P, _P, _P, _P, _P, _SZ, _P]),
    "kvp_keydiff_score": (ctypes.c_int, [_PP, _P, _P, _P, _SZ, _P]),
    "kvp_keydiff_compress": (ctypes.c_int, [_PP, _P, _P, _P, _P, _P, _P, _P, _SZ, _P]),
    "kvp_scores_select": (ctypes.c_int, [_PP, _P, ctypes.POINTER(ctypes.c_int64), _P, _P, _SZ, _P]),
    "kvp_scores_compress_rerotate": (
        ctypes.c_int, [_PP, _P, ctypes.POINTER(ctypes.c_int64), _P, _P, _P, _P, _P, _P, _P, _SZ, _P]),
    "kvp_criticalkv_score": (ctypes.c_int, [_PP, _P, _P, _PI64, _P, _I, _I64, ctypes.c_float, _I, _P, _P, _SZ, _P]),
    "kvp_criticalkv_compress": (
        ctypes.c_int, [_PP, _P, _P, _P, _PI64, _P, _I, _I64, ctypes.c_float, _I, _P, _P, _P, _P, _P, _SZ, _P]),
    "kvp_observed_attention_score": (ctypes.c_int, [_PP, _P, _P, _I, ctypes.c_float, _P, _P, _SZ, _P]),
    "kvp_observed_attention_compress": (
        ctypes.c_int, [_PP, _P, _P, _P, _I, ctypes.c_float, _P, _P, _P, _P, _P, _SZ, _P]),
    "kvp_non_causal_attention_score": (ctypes.c_int, [_PP, _P, _P, _P, _I, _P, _P, _SZ, _P]),
    "kvp_non_causal_attention_compress": (ctypes.c_int, [_PP, _P, _P, _P, _I, _P, _P, _P, _P, _P, _SZ, _P]),
    "kvp_lagkv_score": (ctypes.c_int, [_PP, _P, _P, _I, _I, _I, _P, _P, _SZ, _P]),
    "kvp_lagkv_compress": (ctypes.c_int, [_PP, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _SZ, _P]),
    "kvp_cur_score": (ctypes.c_int, [_PP, _P, _P, _I, _I, _I, _P, _I, _P, _P, _SZ, _P]),
    "kvp_cur_compress": (ctypes.c_int, [_PP, _P, _P, _I, _I, _I, _P, _I, _P, _P, _P, _P, _P, _SZ, _P]),
    "kvp_merging_compress": (
        ctypes.c_int, [_PP, _P, _PI64, _P, _P, ctypes.c_float, ctypes.c_double, _P, _P, _P, _P, _P, _P, _SZ, _P]),
    "kvp_merging_merge": (ctypes.c_int, [_PP, _P, _P, _P, ctypes.c_float, ctypes.c_double, _P, _P, _P, _P, _SZ, _P]),
    "kvp_think_prune": (ctypes.c_int, [_PP, _P, _P, _I, _I, _P, _P, _P, _SZ, _P]),
    "kvp_finch_score": (ctypes.c_int, [_PP, _P, _P, _I, _I, _P, _P, _SZ, _P]),
    "kvp_finch_compress": (ctypes.c_int, [_PP, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P, _SZ, _P]),
    "kvp_scores_compress_chunked": (ctypes.c_int, [_PP, _P, _PI64, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _SZ, _P]),
    "kvp_cam_compress": (
        ctypes.c_int, [_PP, _P, _PI64, _P, _P, _P, _PI64, _I, _I, _P, _P, _P, _P, _PI64, _P, _P, _P, _P, _SZ, _P]),
    "kvp_kvzap_score": (ctypes.c_int, [_PP, _P, _PI64, _I, _I, _P, _P, _P, _P, _P, _P, _SZ, _P]),
    "kvp_kvzap_compress": (
        ctypes.c_int, [_PP, _P, _PI64, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _SZ, _P]),
    "kvp_threshold_evict": (
        ctypes.c_int, [_I, _I, _I, _I, _P, _PI64, _I, ctypes.c_float, _I64, _P, _P, _P, _P, _P, _SZ, _P]),
}

_lib: Optional[ctypes.CDLL] = None


def library_path() -> Path:
    return Path(os.environ.get("KVPRESS_B200_LIB", _LIB_PATH))


def load() -> ctypes.CDLL:
    """Load the shared library (once) and bind every declared symbol. Raises if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    path = library_path()
    if not path.exists():
        raise NativeLibraryError(
            f"{path} not found: build it with `python -m kvpress_b200.build` (needs nvcc). "
            "kvpress_b200 has no CPU or PyTorch fallback."
        )
    lib = ctypes.CDLL(str(path))
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if a declared symbol is not exported
        fn.restype = restype
        fn.argtypes = argtypes
    if lib.kvp_abi_version() != 1:
        raise NativeLibraryError(f"ABI version mismatch: library reports {lib.kvp_abi_version()}")
    _lib = lib
    return lib


def _check(rc: int, what: str) -> None:
    if rc != 0:
        lib = load()
        msg = lib.kvp_status_string(rc).decode()
        if rc == -6:
            msg += ": " + lib.kvp_last_cuda_error().decode()
        raise RuntimeError(f"{what} failed: {msg} (status {rc})")


def _pinned_ok(t: torch.Tensor) -> bool:
    """A pinned host tensor is addressable from the device (UVA): kernels may gather its rows over PCIe."""
    return (not t.is_cuda) and t.is_pinned() and torch.cuda.is_available()


def _require_cuda_kv(keys: torch.Tensor, values: torch.Tensor, pinned_values: bool = False,
                     pinned_keys: bool = False) -> None:
    k_ok = keys.is_cuda or (pinned_keys and _pinned_ok(keys))
    v_ok = values.is_cuda or (pinned_values and _pinned_ok(values))
    if not (k_ok and v_ok):
        raise RuntimeError(
            "kvpress_b200 runs on CUDA tensors only (sm_90a kernels); got "
            f"keys on {keys.device}, values on {values.device}. There is no CPU path."
        )
    if keys.dtype not in _DTYPES or values.dtype != keys.dtype:
        raise RuntimeError(f"kvpress_b200 supports bf16/fp16 caches, got {keys.dtype}/{values.dtype}")
    if keys.dim() != 4 or values.shape != keys.shape:
        raise RuntimeError(f"expected K, V of shape [B, Hkv, S, D], got {tuple(keys.shape)}, {tuple(values.shape)}")


def _out_device(keys: torch.Tensor) -> torch.device:
    return keys.device if keys.is_cuda else torch.device("cuda", torch.cuda.current_device())


def _rows_ok(t: torch.Tensor) -> bool:
    if t.stride(3) != 1 or t.data_ptr() % 16:
        return False
    for dim in range(3):
        if t.shape[dim] > 1 and (t.stride(dim) % 8 or t.stride(dim) < 0):
            return False
    return t.shape[2] == 1 or t.stride(2) >= t.shape[3]


def _normalise(t: torch.Tensor) -> torch.Tensor:
    """Strided views are consumed as they are; only layouts the kernels cannot address are copied."""
    if _rows_ok(t):
        return t
    if not t.is_cuda:
        raise RuntimeError("a pinned host K/V view must already have 16-byte aligned, unit-stride rows")
    return t.contiguous()


def _strides(t: torch.Tensor):
    return tuple(int(t.stride(d)) if t.shape[d] > 1 else 0 for d in range(3))


_PROBLEMS: dict = {}


def make_problem(keys: torch.Tensor, values: torch.Tensor, n_kept: int, num_q_heads: Optional[int] = None) -> KvpProblem:
    """kvp_problem of one call. Structs are cached per (shape, strides, n_kept, Hq, dtype) and must be treated
    as read-only by callers: DecodingPress / per-layer hooks repeat the same few problems thousands of times."""
    key = (keys.shape, keys.stride(), values.stride(), int(n_kept), num_q_heads, keys.dtype)
    p = _PROBLEMS.get(key)
    if p is None:
        p = _build_problem(keys, values, n_kept, num_q_heads)
        if len(_PROBLEMS) > 1024:
            _PROBLEMS.clear()
        _PROBLEMS[key] = p
    return p


def _build_problem(keys: torch.Tensor, values: torch.Tensor, n_kept: int, num_q_heads: Optional[int] = None) -> KvpProblem:
    B, H, S, D = keys.shape
    p = KvpProblem()
    p.B, p.Hkv, p.S, p.D = B, H, S, D
    p.Hq = int(num_q_heads) if num_q_heads else H
    p.n_kept = int(n_kept)
    p.dtype = _DTYPES[keys.dtype]
    ks, vs = _strides(keys), _strides(values)
    # a row stride of 0 only happens for S == 1; keep it addressable
    p.k_stride = (ctypes.c_int64 * 3)(ks[0], ks[1], ks[2] if S > 1 else D)
    p.v_stride = (ctypes.c_int64 * 3)(vs[0], vs[1], vs[2] if S > 1 else D)
    return p


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)


def _stream() -> int:
    """cudaStream_t of torch's current stream on the current device, as an integer handle."""
    if _raw_stream is not None:
        return _raw_stream(torch.cuda.current_device())
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> int:
    """Raw address (0 = NULL); ctypes converts ints to void* through the declared argtypes."""
    return 0 if t is None else t.data_ptr()


_NO_GUARD = contextlib.nullcontext()


def _guard(device: torch.device):
    """Device guard only when the tensor's device is not the current one (the common per-layer hook call
    skips the set-device round trip)."""
    if device.type != "cuda" or device.index is None or device.index == torch.cuda.current_device():
        return _NO_GUARD
    return torch.cuda.device(device)


_WS_BYTES: dict = {}


def workspace_bytes(p: KvpProblem, scorer: int) -> int:
    """kvp_workspace_bytes, asked once per (shape, scorer)."""
    key = (p.B, p.Hkv, p.Hq, p.S, p.D, p.dtype, scorer)
    n = _WS_BYTES.get(key)
    if n is None:
        out = _SZ(0)
        _check(load().kvp_workspace_bytes(ctypes.byref(p), scorer, ctypes.byref(out)), "kvp_workspace_bytes")
        n = _WS_BYTES[key] = int(out.value)
        if len(_WS_BYTES) > 4096:
            _WS_BYTES.clear()
    return n


def launches_per_compress(p: KvpProblem, scorer: int) -> int:
    out = ctypes.c_int(0)
    _check(load().kvp_launches_per_compress(ctypes.byref(p), scorer, ctypes.byref(out)), "kvp_launches_per_compress")
    return int(out.value)


_WS_CACHE: dict = {}


def _workspace(p: KvpProblem, scorer: int, device) -> torch.Tensor:
    """Scratch for one call. Calls on one stream execute in order, so one grow-only buffer per (device, stream)
    is reused instead of allocated per call; under CUDA-graph capture a fresh buffer from the graph's pool is
    used (it must live exactly as long as the graph)."""
    need = workspace_bytes(p, scorer)
    if device.type != "cuda":
        return torch.empty(need, dtype=torch.uint8, device=device)
    if torch.cuda.is_current_stream_capturing():
        return torch.empty(need, dtype=torch.uint8, device=device)
    key = (device.index, _stream())
    ws = _WS_CACHE.get(key)
    if ws is None or ws.numel() < need:
        if len(_WS_CACHE) > 64:
            _WS_CACHE.clear()
        ws = _WS_CACHE[key] = torch.empty(max(need, 1 << 20), dtype=torch.uint8, device=device)
    return ws


# --------------------------------------------------------------------------------------------------
# captured calls: one compress call bound to fixed tensors, replayed as ONE graph launch
# --------------------------------------------------------------------------------------------------
class GraphedCall:
    """`fn()` (any sequence of native.* calls on fixed input tensors) captured into a CUDA graph.

    The C-ABI calls only enqueue kernels / memset nodes on the current stream, never synchronise and never
    allocate, so they are capturable as they are. `replay()` costs one cudaGraphLaunch on the host instead of
    1-6 launches + their argument marshalling: it makes the call GPU-bound on any host (DecodingPress
    compactions, repeated same-shape prefill layers, bench.py). Outputs are the tensors `fn` returned; they are
    overwritten by every replay. The inputs must stay alive and at the same addresses (update them in place)."""

    def __init__(self, fn, warmup: int = 2):
        if not torch.cuda.is_available():
            raise RuntimeError("GraphedCall needs a CUDA device")
        self._fn = fn
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):  # warm-up off the capture: lazy inits (func attributes, ...)
            for _ in range(max(1, warmup)):
                fn()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.outputs = fn()

    def replay(self):
        self.graph.replay()
        return self.outputs

    __call__ = replay


def capture(fn, warmup: int = 2) -> GraphedCall:
    return GraphedCall(fn, warmup)


def workspace_check(p: KvpProblem, scorer: int, workspace: torch.Tensor) -> None:
    """Raises if a kernel of the last call on this workspace abandoned a bounded wait (kvp_workspace_check;
    synchronises the current stream). Debugging aid: the wait only expires on a library bug."""
    _check(load().kvp_workspace_check(ctypes.byref(p), scorer, _ptr(workspace), workspace.numel(), _stream()),
           "kvp_workspace_check")


def _enqueue(name: str, device: torch.device, p: KvpProblem, *args, scorer: Optional[int] = None) -> None:
    """Enqueues the C-ABI call `name` as (p, *args, [workspace, its bytes,] stream) on the current stream of `device`.
    Tensors and None in `args` are passed as addresses; `scorer` names the workspace of a call that takes one."""
    args = [_ptr(a) if a is None or isinstance(a, torch.Tensor) else a for a in args]
    with _guard(device):
        if scorer is not None:
            ws = _workspace(p, scorer, device)
            args += [_ptr(ws), ws.numel()]
        _check(getattr(load(), name)(ctypes.byref(p), *args, _stream()), name)


def _score(name: str, scorer: Optional[int], keys: torch.Tensor, p: KvpProblem, *inputs) -> torch.Tensor:
    """Scores [B, Hkv, S] of a score call (p, *inputs, scores[, workspace], stream)."""
    scores = torch.empty(keys.shape[:3], dtype=keys.dtype, device=keys.device)
    _enqueue(name, keys.device, p, *inputs, scores, scorer=scorer)
    return scores


def _compress(name: str, scorer: Optional[int], keys: torch.Tensor, values: torch.Tensor, n_kept: int, inputs: tuple,
              return_indices: bool, return_scores: Optional[bool] = None, num_q_heads: Optional[int] = None):
    """Outputs of a compress call (p, *inputs, K_out, V_out, idx[, scores][, workspace], stream), enqueued unless
    n_kept == 0: (k_out, v_out, idx, scores), or (k_out, v_out, idx) for a call without a scores output
    (return_scores None). The outputs' device guards the call: pinned host keys have none."""
    p = make_problem(keys, values, n_kept, num_q_heads)
    B, H, S, D = keys.shape
    dev = _out_device(keys)
    k_out = torch.empty((B, H, n_kept, D), dtype=keys.dtype, device=dev)
    v_out = torch.empty_like(k_out)
    idx = torch.empty((B, H, n_kept), dtype=torch.int32, device=dev) if return_indices else None
    outs = (k_out, v_out, idx)
    if return_scores is not None:
        outs += (torch.empty((B, H, S), dtype=keys.dtype, device=dev) if return_scores else None,)
    if n_kept > 0:
        _enqueue(name, dev, p, *inputs, *outs, scorer=scorer)
    return outs


# --------------------------------------------------------------------------------------------------
# Knorm
# --------------------------------------------------------------------------------------------------
def knorm_score(keys: torch.Tensor) -> torch.Tensor:
    _require_cuda_kv(keys, keys)
    keys = _normalise(keys)
    return _score("kvp_knorm_score", None, keys, make_problem(keys, keys, 0), keys)


def knorm_compress(keys, values, n_kept: int, return_indices: bool = False, return_scores: bool = False,
                   _pinned_values: bool = False):
    _require_cuda_kv(keys, values, pinned_values=_pinned_values)
    keys, values = _normalise(keys), _normalise(values)
    return _compress("kvp_knorm_compress", SCORER_KNORM, keys, values, n_kept, (keys, values), return_indices,
                     return_scores)


# --------------------------------------------------------------------------------------------------
# KeyDiff
# --------------------------------------------------------------------------------------------------
def keydiff_score(keys: torch.Tensor) -> torch.Tensor:
    _require_cuda_kv(keys, keys)
    keys = _normalise(keys)
    return _score("kvp_keydiff_score", SCORER_KEYDIFF, keys, make_problem(keys, keys, 0), keys)


def keydiff_compress(keys, values, n_kept: int, return_indices: bool = False, return_scores: bool = False,
                     _pinned_values: bool = False):
    _require_cuda_kv(keys, values, pinned_values=_pinned_values)
    keys, values = _normalise(keys), _normalise(values)
    return _compress("kvp_keydiff_compress", SCORER_KEYDIFF, keys, values, n_kept, (keys, values), return_indices,
                     return_scores)


# --------------------------------------------------------------------------------------------------
# StreamingLLM
# --------------------------------------------------------------------------------------------------
def streaming_score(keys: torch.Tensor, n_kept: int, n_sink: int) -> torch.Tensor:
    _require_cuda_kv(keys, keys)
    return _score("kvp_streaming_score", None, keys, make_problem(keys, keys, n_kept), n_sink)


def streaming_compress(keys, values, n_kept: int, n_sink: int, return_indices: bool = False,
                       _pinned_kv: bool = False):
    _require_cuda_kv(keys, values, pinned_values=_pinned_kv, pinned_keys=_pinned_kv)
    keys, values = _normalise(keys), _normalise(values)
    return _compress("kvp_streaming_compress", None, keys, values, n_kept, (n_sink, keys, values), return_indices)


# --------------------------------------------------------------------------------------------------
# SnapKV
# --------------------------------------------------------------------------------------------------
def _check_q(q_window: torch.Tensor, keys: torch.Tensor, window: int):
    B, _, _, D = keys.shape
    if q_window.dim() != 4 or q_window.shape[0] != B or q_window.shape[2] != window or q_window.shape[3] != D:
        raise RuntimeError(f"q_window must be [B, Hq, {window}, {D}], got {tuple(q_window.shape)}")
    if q_window.dtype != keys.dtype or q_window.device != keys.device:
        raise RuntimeError("q_window must share dtype and device with the keys")
    return q_window.contiguous()


def snapkv_score(keys, q_window, window: int, kernel_size: int) -> torch.Tensor:
    _require_cuda_kv(keys, keys)
    keys = _normalise(keys)
    q_window = _check_q(q_window, keys, window)
    p = make_problem(keys, keys, 0, q_window.shape[1])
    return _score("kvp_snapkv_score", SCORER_SNAPKV, keys, p, keys, q_window, window, kernel_size)


def snapkv_compress(keys, values, q_window, window: int, kernel_size: int, n_kept: int,
                    return_indices: bool = False, return_scores: bool = False, _pinned_values: bool = False):
    _require_cuda_kv(keys, values, pinned_values=_pinned_values)
    keys, values = _normalise(keys), _normalise(values)
    q_window = _check_q(q_window, keys, window)
    return _compress("kvp_snapkv_compress", SCORER_SNAPKV, keys, values, n_kept,
                     (keys, values, q_window, window, kernel_size), return_indices, return_scores, q_window.shape[1])


# --------------------------------------------------------------------------------------------------
# ExpectedAttention
# --------------------------------------------------------------------------------------------------
def _check_stats(mu, cov, keys):
    B, _, _, D = keys.shape
    if mu.dim() != 3 or mu.shape[0] != B or mu.shape[2] != D:
        raise RuntimeError(f"mu must be [B, Hq, {D}], got {tuple(mu.shape)}")
    mu = mu.to(keys.dtype).contiguous()
    if cov is not None:
        if tuple(cov.shape) != (B, mu.shape[1], D, D):
            raise RuntimeError(f"cov must be [B, Hq, {D}, {D}], got {tuple(cov.shape)}")
        cov = cov.to(keys.dtype).contiguous()
    return mu, cov


def expected_attention_score(keys, values, mu, cov, epsilon: float, n_sink: int, use_vnorm: bool) -> torch.Tensor:
    _require_cuda_kv(keys, values)
    keys, values = _normalise(keys), _normalise(values)
    mu, cov = _check_stats(mu, cov, keys)
    p = make_problem(keys, values, 0, mu.shape[1])
    return _score("kvp_expected_attention_score", SCORER_EXPECTED_ATTENTION, keys, p, keys, values, mu, cov,
                  float(epsilon), n_sink, int(bool(use_vnorm)))


def expected_attention_compress(keys, values, mu, cov, epsilon: float, n_sink: int, use_vnorm: bool, n_kept: int,
                                return_indices: bool = False, return_scores: bool = False):
    _require_cuda_kv(keys, values)
    keys, values = _normalise(keys), _normalise(values)
    mu, cov = _check_stats(mu, cov, keys)
    return _compress("kvp_expected_attention_compress", SCORER_EXPECTED_ATTENTION, keys, values, n_kept,
                     (keys, values, mu, cov, float(epsilon), n_sink, int(bool(use_vnorm))), return_indices,
                     return_scores, mu.shape[1])


# --------------------------------------------------------------------------------------------------
# generic scores (wrapper presses, user-defined ScorerPress subclasses)
# --------------------------------------------------------------------------------------------------
def _unit_stride_scores(scores: torch.Tensor):
    """[B, H, S] scores with unit stride along S (copied only when needed) and their (b, h) element strides for the
    C ABI, 0 along a dim of size 1."""
    if scores.stride(2) != 1:
        scores = scores.contiguous()
    return scores, (ctypes.c_int64 * 2)(*(scores.stride(d) if scores.shape[d] > 1 else 0 for d in range(2)))


def _caller_scores(scores: torch.Tensor, keys: torch.Tensor):
    """Caller-supplied scores of the cache `keys`, checked and cast to its dtype; see _unit_stride_scores."""
    if tuple(scores.shape) != tuple(keys.shape[:3]) or scores.device != keys.device:
        raise RuntimeError(f"scores must be [B, Hkv, S] on the cache device, got {tuple(scores.shape)}")
    return _unit_stride_scores(scores.to(keys.dtype))


def scores_compress(scores: torch.Tensor, keys, values, n_kept: int, return_indices: bool = False):
    """Top-k + compaction for caller-supplied scores [B, Hkv, S] (wrapper presses, user ScorerPress subclasses).

    The selection kernels rank 16-bit keys: scores are compared IN THE CACHE DTYPE. The in-scope scorers return that
    dtype already (as the reference's do); fp32 scores of a custom press are rounded to it first, so values that
    differ only below bf16 / fp16 resolution become ties and go to the lowest positions, where the reference's fp32
    `topk` would still order them."""
    _require_cuda_kv(keys, values)
    keys, values = _normalise(keys), _normalise(values)
    scores, sstride = _caller_scores(scores, keys)
    return _compress("kvp_scores_compress", SCORER_GENERIC, keys, values, n_kept, (scores, sstride, keys, values),
                     return_indices)


def scores_select(scores: torch.Tensor, n_kept: int) -> torch.Tensor:
    """Positions of the n_kept largest scores of every row of a [B, H, S] bf16/fp16 CUDA tensor, ascending
    (ties to the lowest positions), int32 [B, H, n_kept]. No K/V involved."""
    if not scores.is_cuda or scores.dtype not in _DTYPES or scores.dim() != 3:
        raise RuntimeError(f"scores must be a CUDA bf16/fp16 [B, H, S] tensor, got {scores.dtype} on {scores.device}")
    scores, sstride = _unit_stride_scores(scores)
    B, H, S = scores.shape
    p = KvpProblem()
    p.B, p.Hkv, p.Hq, p.S, p.D, p.n_kept, p.dtype = B, H, H, S, 8, int(n_kept), _DTYPES[scores.dtype]
    idx = torch.empty((B, H, n_kept), dtype=torch.int32, device=scores.device)
    if n_kept > 0:
        _enqueue("kvp_scores_select", scores.device, p, scores, sstride, idx, scorer=SCORER_GENERIC)
    return idx


def scores_compress_rerotate(scores: torch.Tensor, keys, values, n_kept: int, inv_freq: torch.Tensor,
                             return_indices: bool = False):
    """KeyRerotationPress: top-k + compaction with the kept keys re-rotated to their new positions."""
    _require_cuda_kv(keys, values)
    keys, values = _normalise(keys), _normalise(values)
    scores, sstride = _caller_scores(scores, keys)
    if inv_freq.numel() * 2 != keys.shape[3]:
        raise RuntimeError(f"inv_freq must have head_dim/2 = {keys.shape[3] // 2} entries, got {inv_freq.numel()}")
    inv_freq = inv_freq.to(device=keys.device, dtype=torch.float32).contiguous()
    return _compress("kvp_scores_compress_rerotate", SCORER_GENERIC, keys, values, n_kept,
                     (scores, sstride, keys, values, inv_freq), return_indices)


# --------------------------------------------------------------------------------------------------
# CriticalKV (on the scores of the press it wraps)
# --------------------------------------------------------------------------------------------------
def _check_wo(wo: torch.Tensor, values: torch.Tensor):
    """o_proj.weight [hidden, Hq*D] in the cache dtype with unit-stride rows: (wo, Hq, row stride). Sliced rows are
    consumed in place; a layout the kernel cannot address is copied."""
    D = values.shape[3]
    if wo.dim() != 2 or wo.shape[1] % D or wo.device != values.device:
        raise RuntimeError(f"wo must be o_proj.weight [hidden, Hq*{D}] on the cache device, got {tuple(wo.shape)}")
    wo = wo.to(values.dtype)
    if wo.stride(1) != 1 or wo.data_ptr() % 16 or (wo.shape[0] > 1 and wo.stride(0) % 8):
        wo = wo.contiguous()
    return wo, wo.shape[1] // D, int(wo.stride(0) if wo.shape[0] > 1 else wo.shape[1])


def criticalkv_score(base_scores: torch.Tensor, values: torch.Tensor, wo: torch.Tensor, epsilon: float,
                     n_first: int) -> torch.Tensor:
    """CriticalKV scores [B, Hkv, S] from the wrapped press's scores: (base + epsilon) * the mean over the group of
    ||v_s Wo_h^T||_1, then finfo.max on the n_first best base scores of every row."""
    _require_cuda_kv(values, values)
    values = _normalise(values)
    wo, Hq, wo_stride = _check_wo(wo, values)
    base, sstride = _caller_scores(base_scores, values)
    p = make_problem(values, values, 0, Hq)
    return _score("kvp_criticalkv_score", SCORER_CRITICALKV, values, p, values, base, sstride, wo, wo.shape[0],
                  wo_stride, float(epsilon), int(n_first))


def criticalkv_compress(base_scores: torch.Tensor, keys, values, wo: torch.Tensor, epsilon: float, n_first: int,
                        n_kept: int, return_indices: bool = False, return_scores: bool = False):
    """criticalkv_score, then top-n_kept + compaction on the final scores."""
    _require_cuda_kv(keys, values)
    keys, values = _normalise(keys), _normalise(values)
    wo, Hq, wo_stride = _check_wo(wo, values)
    base, sstride = _caller_scores(base_scores, keys)
    return _compress("kvp_criticalkv_compress", SCORER_CRITICALKV, keys, values, n_kept,
                     (keys, values, base, sstride, wo, wo.shape[0], wo_stride, float(epsilon), int(n_first)),
                     return_indices, return_scores, Hq)


# --------------------------------------------------------------------------------------------------
# ObservedAttention (H2O)
# --------------------------------------------------------------------------------------------------
def _check_queries(q: torch.Tensor, keys: torch.Tensor) -> torch.Tensor:
    """RoPE'd queries [B, Hq, n_q, D] with 1 <= n_q <= S, in the cache dtype and on its device, made contiguous."""
    B, _, S, D = keys.shape
    if q.dim() != 4 or q.shape[0] != B or q.shape[3] != D or not 1 <= q.shape[2] <= S:
        raise RuntimeError(f"q must be [B, Hq, n_q, {D}] with 1 <= n_q <= {S}, got {tuple(q.shape)}")
    if q.dtype != keys.dtype or q.device != keys.device:
        raise RuntimeError("q must share dtype and device with the keys")
    return q.contiguous()


def observed_attention_score(keys, q, scaling: float) -> torch.Tensor:
    """H2O scores [B, Hkv, S]: the causal softmax(scaling q.k) of the n_q queries q [B, Hq, n_q, D] (the last n_q
    positions), summed over the queries, divided by S - s in the cache dtype, averaged over the group."""
    _require_cuda_kv(keys, keys)
    keys = _normalise(keys)
    q = _check_queries(q, keys)
    p = make_problem(keys, keys, 0, q.shape[1])
    return _score("kvp_observed_attention_score", SCORER_OBSERVED_ATTENTION, keys, p, keys, q, q.shape[2],
                  float(scaling))


def observed_attention_compress(keys, values, q, scaling: float, n_kept: int, return_indices: bool = False,
                                return_scores: bool = False):
    """observed_attention_score, then top-n_kept + compaction."""
    _require_cuda_kv(keys, values)
    keys, values = _normalise(keys), _normalise(values)
    q = _check_queries(q, keys)
    return _compress("kvp_observed_attention_compress", SCORER_OBSERVED_ATTENTION, keys, values, n_kept,
                     (keys, values, q, q.shape[2], float(scaling)), return_indices, return_scores, q.shape[1])


# --------------------------------------------------------------------------------------------------
# NonCausalAttention (the attention half of Compactor)
# --------------------------------------------------------------------------------------------------
def _check_prefill_queries(q: torch.Tensor, keys: torch.Tensor) -> torch.Tensor:
    """RoPE'd queries [B, Hq, S, D] of every cached position, in the cache dtype and on its device, made contiguous."""
    B, _, S, D = keys.shape
    if q.dim() != 4 or q.shape[0] != B or q.shape[2] != S or q.shape[3] != D:
        raise RuntimeError(f"q must be [B, Hq, {S}, {D}] (prefill: one query per cached position), got {tuple(q.shape)}")
    if q.dtype != keys.dtype or q.device != keys.device:
        raise RuntimeError("q must share dtype and device with the keys")
    return q.contiguous()


def non_causal_attention_score(keys, values, q, chunk_size: int) -> torch.Tensor:
    """NonCausalAttnPress scores [B, Hkv, S]: the chunked non-causal softmax(q.k) (no scaling) summed over each chunk's
    queries, averaged over the group, times ||v||, pooled over 3 positions and z-normalised over the whole tensor."""
    _require_cuda_kv(keys, values)
    keys, values = _normalise(keys), _normalise(values)
    q = _check_prefill_queries(q, keys)
    p = make_problem(keys, values, 0, q.shape[1])
    return _score("kvp_non_causal_attention_score", SCORER_NON_CAUSAL_ATTENTION, keys, p, keys, values, q,
                  int(chunk_size))


def non_causal_attention_compress(keys, values, q, chunk_size: int, n_kept: int, return_indices: bool = False,
                                  return_scores: bool = False):
    """non_causal_attention_score, then top-n_kept + compaction."""
    _require_cuda_kv(keys, values)
    keys, values = _normalise(keys), _normalise(values)
    q = _check_prefill_queries(q, keys)
    return _compress("kvp_non_causal_attention_compress", SCORER_NON_CAUSAL_ATTENTION, keys, values, n_kept,
                     (keys, values, q, int(chunk_size)), return_indices, return_scores, q.shape[1])


# --------------------------------------------------------------------------------------------------
# LagKV
# --------------------------------------------------------------------------------------------------
def lagkv_score(keys, values, n_sink: int, lag_size: int, cross_scoring: bool) -> torch.Tensor:
    """LagKVPress scores [B, Hkv, S] (include/kvpress_b200.h, kvp_lagkv_score): per partition of lag_size positions, the
    softmax of the std of the keys and values scaled by the next partition's min / max, as ranks / lag_size, or the
    averaged softmax itself with cross_scoring; the sinks and the tail score 1."""
    _require_cuda_kv(keys, values)
    keys, values = _normalise(keys), _normalise(values)
    return _score("kvp_lagkv_score", SCORER_LAGKV, keys, make_problem(keys, values, 0), keys, values, int(n_sink),
                  int(lag_size), int(bool(cross_scoring)))


def lagkv_compress(keys, values, n_sink: int, lag_size: int, cross_scoring: bool, n_kept: int,
                   return_indices: bool = False, return_scores: bool = False):
    """lagkv_score, then top-n_kept + compaction."""
    _require_cuda_kv(keys, values)
    keys, values = _normalise(keys), _normalise(values)
    return _compress("kvp_lagkv_compress", SCORER_LAGKV, keys, values, n_kept,
                     (keys, values, int(n_sink), int(lag_size), int(bool(cross_scoring))), return_indices,
                     return_scores)


# --------------------------------------------------------------------------------------------------
# CUR
# --------------------------------------------------------------------------------------------------
def _cur_inputs(keys, values, num_sinks: int, leverage_type: str, local_window_size: int, G) -> tuple:
    """The arguments of kvp_cur_score / kvp_cur_compress between the kvp_problem and the outputs."""
    if leverage_type not in CUR_LEVERAGE_TYPES:
        raise ValueError("Unknown leverage type: choose from 'kv_avg', 'key', 'value' or 'kv_product'")
    r = 0
    if G is not None:
        if G.dtype != torch.float32 or G.dim() != 2 or G.shape[0] != keys.shape[-1] or G.device != keys.device:
            raise RuntimeError(f"expected a float32 projection [head_dim, r] on {keys.device}, got "
                               f"{G.dtype} {tuple(G.shape)} on {G.device}")
        G, r = G.contiguous(), G.shape[1]
    return keys, values, int(num_sinks), CUR_LEVERAGE_TYPES.index(leverage_type), int(local_window_size), G, int(r)


def cur_score(keys, values, num_sinks: int, leverage_type: str, local_window_size: int, G=None) -> torch.Tensor:
    """CURPress scores [B, Hkv, S] (include/kvpress_b200.h, kvp_cur_score): the squared norms of the keys and of the
    values (of their projections by G [D, r], float32, when given), each divided by its sum over its window of
    local_window_size positions (0: not divided), combined by leverage_type, divided by the row's sum; the first
    num_sinks positions score 1."""
    _require_cuda_kv(keys, values)
    keys, values = _normalise(keys), _normalise(values)
    inputs = _cur_inputs(keys, values, num_sinks, leverage_type, local_window_size, G)
    return _score("kvp_cur_score", SCORER_CUR, keys, make_problem(keys, values, 0), *inputs)


def cur_compress(keys, values, num_sinks: int, leverage_type: str, local_window_size: int, G, n_kept: int,
                 return_indices: bool = False, return_scores: bool = False):
    """cur_score, then top-n_kept + compaction."""
    _require_cuda_kv(keys, values)
    keys, values = _normalise(keys), _normalise(values)
    inputs = _cur_inputs(keys, values, num_sinks, leverage_type, local_window_size, G)
    return _compress("kvp_cur_compress", SCORER_CUR, keys, values, n_kept, inputs, return_indices, return_scores)


# --------------------------------------------------------------------------------------------------
# Merging (MergingPress: evicted values folded into their most cosine-similar kept row)
# --------------------------------------------------------------------------------------------------
def _merging_gate(similarity_threshold: float, merge_fraction: float) -> tuple:
    if not 0.0 <= similarity_threshold <= 1.0:
        raise ValueError(f"similarity_threshold must be in [0, 1], got {similarity_threshold}")
    if not 0.0 < merge_fraction <= 1.0:
        raise ValueError(f"merge_fraction must be in (0, 1], got {merge_fraction}")
    return float(similarity_threshold), float(merge_fraction)


def _merge_plan(keys: torch.Tensor, dev, n_evict: int, return_plan: bool):
    """target_out / sim_out of a merging call: int32 and float32 [B, Hkv, n_evict], or None."""
    if not return_plan:
        return None, None
    shape = (*keys.shape[:2], n_evict)
    return (torch.empty(shape, dtype=torch.int32, device=dev), torch.empty(shape, dtype=torch.float32, device=dev))


def merging_compress(scores: torch.Tensor, keys, values, similarity_threshold: float, merge_fraction: float,
                     n_kept: int, return_indices: bool = False, return_plan: bool = False):
    """MergingPress.compress (include/kvpress_b200.h, kvp_merging_compress): the n_kept best `scores` of every row are
    kept, as scores_compress keeps them, and every evicted value is first folded into the kept row whose key is most
    cosine-similar. Returns (k_out, v_out, idx, target, sim): idx with return_indices, and with return_plan the merge
    plan (target in kept-slot numbering, int32, and max_sim, float32, [B, Hkv, S - n_kept]); None otherwise."""
    _require_cuda_kv(keys, values)
    keys, values = _normalise(keys), _normalise(values)
    scores, sstride = _caller_scores(scores, keys)
    thr, frac = _merging_gate(similarity_threshold, merge_fraction)
    B, H, S, D = keys.shape
    dev = keys.device
    k_out = torch.empty((B, H, n_kept, D), dtype=keys.dtype, device=dev)
    v_out = torch.empty_like(k_out)
    idx = torch.empty((B, H, n_kept), dtype=torch.int32, device=dev) if return_indices else None
    target, sim = _merge_plan(keys, dev, S - n_kept, return_plan)
    if n_kept > 0:
        _enqueue("kvp_merging_compress", dev, make_problem(keys, values, n_kept), scores, sstride, keys, values, thr,
                 frac, k_out, v_out, idx, target, sim, scorer=SCORER_MERGING)
    return k_out, v_out, idx, target, sim


def merging_merge(keys, values, kept_idx: torch.Tensor, similarity_threshold: float, merge_fraction: float,
                  return_plan: bool = False):
    """The merge alone (include/kvpress_b200.h, kvp_merging_merge) on caller kept positions kept_idx [B, Hkv, n_kept]
    (ascending and distinct; cast to int32): the merged kept value rows [B, Hkv, n_kept, D], then the merge plan as in
    merging_compress. Returns (v_out, target, sim)."""
    _require_cuda_kv(keys, values)
    keys, values = _normalise(keys), _normalise(values)
    thr, frac = _merging_gate(similarity_threshold, merge_fraction)
    B, H, S, D = keys.shape
    if kept_idx.dim() != 3 or tuple(kept_idx.shape[:2]) != (B, H) or kept_idx.shape[2] > S or kept_idx.device != keys.device:
        raise RuntimeError(f"kept_idx must be [B, Hkv, n_kept <= {S}] on the cache device, got {tuple(kept_idx.shape)}")
    kept_idx = kept_idx.to(torch.int32).contiguous()
    n_kept = kept_idx.shape[2]
    v_out = torch.empty((B, H, n_kept, D), dtype=values.dtype, device=keys.device)
    target, sim = _merge_plan(keys, keys.device, S - n_kept, return_plan)
    _enqueue("kvp_merging_merge", keys.device, make_problem(keys, values, n_kept), keys, values, kept_idx, thr, frac,
             v_out, target, sim, scorer=SCORER_MERGING)
    return v_out, target, sim


# --------------------------------------------------------------------------------------------------
# ThinK (key channels zeroed in place)
# --------------------------------------------------------------------------------------------------
def think_prune(keys: torch.Tensor, q_window: torch.Tensor, n_pruned: int, return_pruned: bool = False,
                return_scores: bool = False):
    """ThinKPress.compress (include/kvpress_b200.h, kvp_think_prune): the n_pruned key channels of every [B, Hkv] row
    with the smallest qn * kn are set to +0 IN PLACE, qn the mean square of the channel over the window queries
    q_window [B, Hq, w, D] of the kv head's query heads, kn its mean square over the cached positions (ties: the higher
    channel is pruned; NaN is pruned last). Returns (keys, pruned, scores): the same keys tensor, and with return_pruned
    the pruned channels ascending (int32 [B, Hkv, n_pruned]), with return_scores the fp32 channel scores [B, Hkv, D].
    With n_pruned == 0 nothing is enqueued and both optional outputs are None."""
    _require_cuda_kv(keys, keys)
    if not _rows_ok(keys):
        raise RuntimeError("think_prune writes the keys in place: they need 16-byte aligned, unit-stride rows with "
                           "outer strides that are multiples of 8 elements")
    B, H, S, D = keys.shape
    if not 0 <= n_pruned <= D:
        raise ValueError(f"n_pruned must be in [0, {D}], got {n_pruned}")
    if q_window.dim() != 4 or q_window.shape[0] != B or q_window.shape[3] != D or q_window.shape[2] < 1 or \
            q_window.shape[1] % H:
        raise RuntimeError(f"q_window must be [B, Hq, w >= 1, {D}] with Hq a multiple of {H}, got {tuple(q_window.shape)}")
    if q_window.dtype != keys.dtype or q_window.device != keys.device:
        raise RuntimeError("q_window must share dtype and device with the keys")
    if n_pruned == 0:
        return keys, None, None
    q_window = q_window.contiguous()
    pruned = torch.empty((B, H, n_pruned), dtype=torch.int32, device=keys.device) if return_pruned else None
    scores = torch.empty((B, H, D), dtype=torch.float32, device=keys.device) if return_scores else None
    _enqueue("kvp_think_prune", keys.device, make_problem(keys, keys, S, q_window.shape[1]), keys, q_window,
             q_window.shape[2], int(n_pruned), pruned, scores, scorer=SCORER_THINK)
    return keys, pruned, scores


# --------------------------------------------------------------------------------------------------
# Finch
# --------------------------------------------------------------------------------------------------
def chunk_counts(S: int, chunk_length: Optional[int], compression_ratio: float):
    """(chunk_length, chunk_kept, tail_kept, n_kept) of FinchPress's selection: chunk_length 0 (None) keeps
    int(S (1 - r)) of the row; otherwise each full chunk keeps max(1, int(L (1 - r))) and the short last chunk
    max(1, int(len (1 - r))), as the reference's loop over chunks does."""
    if not chunk_length:
        return 0, 0, 0, int(S * (1 - compression_ratio))
    L = int(chunk_length)
    n_full, tail = divmod(S, L)
    chunk_kept = max(1, int(L * (1 - compression_ratio))) if n_full else 0
    tail_kept = max(1, int(tail * (1 - compression_ratio))) if tail else 0
    return L, chunk_kept, tail_kept, n_full * chunk_kept + tail_kept


def _inv_freq(inv_freq: Optional[torch.Tensor], keys: torch.Tensor) -> Optional[torch.Tensor]:
    if inv_freq is None:
        return None
    if inv_freq.numel() * 2 != keys.shape[3]:
        raise RuntimeError(f"inv_freq must have head_dim/2 = {keys.shape[3] // 2} entries, got {inv_freq.numel()}")
    return inv_freq.to(device=keys.device, dtype=torch.float32).contiguous()


def finch_score(keys, q_window, window: int, normalize: bool = True) -> torch.Tensor:
    """FinchPress.score (include/kvpress_b200.h, kvp_finch_score): [B, Hkv, S] in the cache dtype, the window
    positions holding the reference's max + 1 sentinel."""
    _require_cuda_kv(keys, keys)
    keys = _normalise(keys)
    q_window = _check_q(q_window, keys, window)
    p = make_problem(keys, keys, 0, q_window.shape[1])
    return _score("kvp_finch_score", SCORER_FINCH, keys, p, keys, q_window, window, int(bool(normalize)))


def finch_compress(keys, values, q_window, window: int, compression_ratio: float, chunk_length: Optional[int] = None,
                   normalize: bool = True, inv_freq: Optional[torch.Tensor] = None, return_indices: bool = False,
                   return_scores: bool = False):
    """FinchPress.compress (kvp_finch_compress): the scores, the per-chunk selection (chunk_length None: the whole
    row) and the compaction, the kept keys re-rotated to their new positions when inv_freq is given.
    Returns (k_out, v_out, idx, scores)."""
    _require_cuda_kv(keys, values)
    keys, values = _normalise(keys), _normalise(values)
    q_window = _check_q(q_window, keys, window)
    L, chunk_kept, tail_kept, n_kept = chunk_counts(keys.shape[2], chunk_length, compression_ratio)
    return _compress("kvp_finch_compress", SCORER_FINCH, keys, values, n_kept,
                     (keys, values, q_window, window, int(bool(normalize)), L, chunk_kept, tail_kept,
                      _inv_freq(inv_freq, keys)), return_indices, return_scores, q_window.shape[1])


def scores_compress_chunked(scores: torch.Tensor, keys, values, compression_ratio: float, chunk_length: int,
                            inv_freq: Optional[torch.Tensor] = None, return_indices: bool = False):
    """FinchPress's chunked selection on caller scores [B, Hkv, S] (kvp_scores_compress_chunked): each chunk of
    chunk_length positions keeps its best max(1, int(len (1 - r))), the kept keys optionally re-rotated to their
    new positions. Returns (k_out, v_out, idx)."""
    _require_cuda_kv(keys, values)
    keys, values = _normalise(keys), _normalise(values)
    scores, sstride = _caller_scores(scores, keys)
    L, chunk_kept, tail_kept, n_kept = chunk_counts(keys.shape[2], chunk_length, compression_ratio)
    if L < 1:
        raise RuntimeError("scores_compress_chunked needs chunk_length >= 1")
    return _compress("kvp_scores_compress_chunked", SCORER_FINCH, keys, values, n_kept,
                     (scores, sstride, L, chunk_kept, tail_kept, keys, values, _inv_freq(inv_freq, keys)),
                     return_indices)


# --------------------------------------------------------------------------------------------------
# CaM (CAMPress: evicted values merged into the kept rows after them, then pruned)
# --------------------------------------------------------------------------------------------------
def _attn_view(a: torch.Tensor, shape: tuple, keys: torch.Tensor, name: str):
    """A float32 [B, Hkv, n] view with unit stride along n (it may sit in a capacity buffer) and its (b, h) strides."""
    if a.dtype != torch.float32 or tuple(a.shape) != shape or a.device != keys.device or (shape[2] > 1 and a.stride(2) != 1):
        raise RuntimeError(f"{name} must be a float32 {list(shape)} view with unit stride along the last dim on "
                           f"{keys.device}, got {a.dtype} {tuple(a.shape)} on {a.device}")
    return (ctypes.c_int64 * 2)(*(a.stride(d) if a.shape[d] > 1 else 0 for d in range(2)))


def cam_compress(scores: torch.Tensor, keys, values, attn_sum: torch.Tensor, attn_out: torch.Tensor, n_merge: int,
                 merge_budget: int, uniforms: Optional[torch.Tensor], n_kept: int, return_indices: bool = False,
                 return_plan: bool = False):
    """CAMPress.compress (include/kvpress_b200.h, kvp_cam_compress): the n_kept best head means of `scores` are kept
    (one selection per batch element), the n_merge best evicted positions are merged, each with probability
    clamp(A[e] / window mean of A), into the merge_budget kept rows after it, and K, V and the running sum attn_sum
    (float32 [B, Hkv, S]) are compacted; the pruned sum is written into attn_out (float32 [B, Hkv, n_kept]). uniforms:
    float32 [B, Hkv, n_merge] in [0, 1), the draws. Returns (k_out, v_out, idx, merge_idx, merge_prob): idx (int32
    [B, n_kept]) with return_indices, and with return_plan the candidates (int32 [B, n_merge]) and their
    probabilities (float32 [B, Hkv, n_merge]); None otherwise."""
    _require_cuda_kv(keys, values)
    keys, values = _normalise(keys), _normalise(values)
    scores, sstride = _caller_scores(scores, keys)
    B, H, S, D = keys.shape
    astride = _attn_view(attn_sum, (B, H, S), keys, "attn_sum")
    ostride = _attn_view(attn_out, (B, H, n_kept), keys, "attn_out")
    if not 0 <= n_merge <= S - n_kept or merge_budget < 1:
        raise ValueError(f"need 0 <= n_merge <= {S - n_kept} and merge_budget >= 1, got {n_merge}, {merge_budget}")
    if n_merge > 0:
        if uniforms is None or tuple(uniforms.shape) != (B, H, n_merge) or uniforms.device != keys.device:
            raise RuntimeError(f"uniforms must be [{B}, {H}, {n_merge}] on {keys.device}")
        uniforms = uniforms.to(torch.float32).contiguous()
    else:
        uniforms = None
    dev = keys.device
    k_out = torch.empty((B, H, n_kept, D), dtype=keys.dtype, device=dev)
    v_out = torch.empty_like(k_out)
    idx = torch.empty((B, n_kept), dtype=torch.int32, device=dev) if return_indices else None
    merge_idx = torch.empty((B, n_merge), dtype=torch.int32, device=dev) if return_plan else None
    merge_prob = torch.empty((B, H, n_merge), dtype=torch.float32, device=dev) if return_plan else None
    if n_kept > 0:
        _enqueue("kvp_cam_compress", dev, make_problem(keys, values, n_kept), scores, sstride, keys, values, attn_sum,
                 astride, int(n_merge), int(merge_budget), uniforms, k_out, v_out, attn_out, ostride, idx, merge_idx,
                 merge_prob, scorer=SCORER_CAM)
    return k_out, v_out, idx, merge_idx, merge_prob


# --------------------------------------------------------------------------------------------------
# KVzap (KVzapPress: a surrogate model of the hidden states) and DMS (DMSPress: threshold eviction)
# --------------------------------------------------------------------------------------------------
def kvzap_supported(hidden: int, hd: int, n_heads: int) -> bool:
    """The shapes kvp_kvzap_* take (include/kvpress_b200.h); KVzapPress scores others with cuBLAS."""
    return (hidden % 8 == 0 and 0 < hidden <= KVZAP_MAX_HIDDEN and hd % 8 == 0 and 0 <= hd <= KVZAP_MAX_HD
            and 0 < n_heads <= KVZAP_MAX_HEADS)


def _kvzap_inputs(hidden_states: torch.Tensor, keys: torch.Tensor, weights: tuple):
    """(x, its (b, s) strides, hidden, hd, w1, b1, w2, b2) of a kvp_kvzap_* call. weights = (w1, b1, w2, b2) in the
    cache dtype on its device (MLP), or (W, b, None, None) (linear)."""
    B, H, S, _ = keys.shape
    x = hidden_states
    if x.dim() != 3 or x.shape[0] != B or x.shape[1] != S or x.dtype != keys.dtype or x.device != keys.device:
        raise RuntimeError(f"hidden_states must be [{B}, {S}, hidden] {keys.dtype} on {keys.device}, got "
                           f"{tuple(x.shape)} {x.dtype} on {x.device}")
    if x.stride(2) != 1 or x.data_ptr() % 16 or any(x.shape[d] > 1 and (x.stride(d) % 8 or x.stride(d) < 0)
                                                    for d in range(2)):
        x = x.contiguous()
    w1, b1, w2, b2 = weights
    hd = 0 if w2 is None else int(w1.shape[0])
    for t in (w1, b1, w2, b2):
        if t is not None and (t.dtype != keys.dtype or t.device != keys.device or not t.is_contiguous()):
            raise RuntimeError(f"KVzap weights must be contiguous {keys.dtype} on {keys.device}")
    xstride = (ctypes.c_int64 * 2)(*(x.stride(d) if x.shape[d] > 1 else 0 for d in range(2)))
    return x, xstride, int(x.shape[2]), hd, w1, b1, w2, b2


def kvzap_score(hidden_states: torch.Tensor, keys: torch.Tensor, values: torch.Tensor, weights: tuple) -> torch.Tensor:
    """KVzapPress.score (kvp_kvzap_score): the surrogate model's scores [B, Hkv, S] in the cache dtype."""
    _require_cuda_kv(keys, values)
    keys, values = _normalise(keys), _normalise(values)
    return _score("kvp_kvzap_score", SCORER_KVZAP, keys, make_problem(keys, values, 0),
                  *_kvzap_inputs(hidden_states, keys, weights))


def kvzap_compress(hidden_states: torch.Tensor, keys, values, weights: tuple, n_kept: int,
                   return_indices: bool = False, return_scores: bool = False):
    """KVzapPress.compress (kvp_kvzap_compress): the scores above, the n_kept best per head, K / V compacted.
    Returns (k_out, v_out, idx, scores)."""
    _require_cuda_kv(keys, values)
    keys, values = _normalise(keys), _normalise(values)
    return _compress("kvp_kvzap_compress", SCORER_KVZAP, keys, values, n_kept,
                     (*_kvzap_inputs(hidden_states, keys, weights), keys, values), return_indices, return_scores)


def threshold_evict(scores: torch.Tensor, n_evict: int, threshold: float, shift: int) -> list:
    """DMSPress's eviction (kvp_threshold_evict): [b, h, s + shift] (int64) of every scores[b, h, s] < threshold with
    s < n_evict, in torch.where order, the threshold rounded to the score dtype as torch does. One host read (the
    count)."""
    if not scores.is_cuda or scores.dtype not in _DTYPES or scores.dim() != 3:
        raise RuntimeError(f"scores must be a CUDA bf16/fp16 [B, Hkv, n] tensor, got {scores.dtype} "
                           f"{tuple(scores.shape)} on {scores.device}")
    B, H, n = scores.shape
    if not 0 <= n_evict <= n:
        raise ValueError(f"need 0 <= n_evict <= {n}, got {n_evict}")
    if n > 1 and scores.stride(2) != 1 or scores.data_ptr() % 2:
        scores = scores.contiguous()
    sstride = (ctypes.c_int64 * 2)(*(scores.stride(d) if scores.shape[d] > 1 else 0 for d in range(2)))
    dev = scores.device
    out = torch.empty((3, B * H * n_evict), dtype=torch.int64, device=dev)
    count = torch.empty((1,), dtype=torch.int64, device=dev)
    ws = torch.empty(((B * H * -(-n // 4096) * 8 + 255) // 256 * 256,), dtype=torch.uint8, device=dev)
    with _guard(dev):
        _check(load().kvp_threshold_evict(_DTYPES[scores.dtype], B, H, n, _ptr(scores), sstride, int(n_evict),
                                          float(threshold), int(shift), _ptr(out[0]), _ptr(out[1]), _ptr(out[2]),
                                          _ptr(count), _ptr(ws), ws.numel(), _stream()), "kvp_threshold_evict")
    c = int(count.item())
    # copies of exactly the count, as torch.where returns: DMSPress keeps them for the rest of the generation
    return list(out[:, :c].clone().unbind(0))
