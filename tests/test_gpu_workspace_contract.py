"""The memory contract of every C-ABI entry point (include/kvpress_b200.h, "Conventions" and kvp_workspace_bytes), on
exact-size, poisoned and shared workspaces with guarded outputs.

Every buffer a call is given lives in its own allocation laid out as [guard | buffer | guard], with 64 KiB guards of a
known byte. The workspace is exactly kvp_workspace_bytes bytes (native._workspace is replaced for the call); the
outputs (scores, K_out, V_out, idx, target, sim) are views of their own arenas; the call is enqueued through
native._enqueue with the argument order of its public wrapper. For every case:
1. the outputs are bitwise equal under every workspace fill (0x00, 0xFF, seeded random bytes) and output fill (0x00,
   0xFF), and bitwise equal to the same call through the public native.* wrapper: an output element no kernel writes,
   or a value read from scratch no kernel wrote first, breaks this;
2. every guard byte, of the workspace and of every output, is unchanged;
3. native.workspace_check reports no expired bounded wait. A call that neither clears the workspace's leading region
   nor waits on it leaves the flag as it found it (the Knorm cluster kernel, the KeyDiff and LagKV score calls, the
   CriticalKV score call without a first stage and the Merging merge call), so it is read after the others only;
4. the inputs are bitwise unchanged;
5. a compress, select or merge call with n_kept == 0 leaves the workspace, the outputs and the guards as they were.
Then: a sequence of calls of every scorer on ONE shared arena (growing and shrinking shapes, the same scorer and shape
twice in a row on new inputs) gives each call's result on a fresh poisoned workspace; calls interleaved on two streams,
and issued from two host threads, each with its own workspace, give their serial results; and a workspace whose base
is 16 mod 256 bytes (the ABI asks only for 16-byte alignment) gives the same results.
"""
import threading
from dataclasses import dataclass
from typing import Callable, Optional

import pytest
import torch

from kvpress_b200 import native as N
from tests.gpu_support import (DEV, _native, ckv_inputs, ea_inputs, lagkv_inputs, nca_inputs, oa_inputs,
                               rope_inv_freq, snap_inputs)

gpu = pytest.mark.gpu
GUARD = 64 << 10
PATTERN = 0xA5
WS_FILLS = ("zeros", "ones", "random")
OUT_FILLS = ("zeros", "ones")
SCORER = dict(generic=N.SCORER_GENERIC, knorm=N.SCORER_KNORM, snapkv=N.SCORER_SNAPKV, ea=N.SCORER_EXPECTED_ATTENTION,
              keydiff=N.SCORER_KEYDIFF, ckv=N.SCORER_CRITICALKV, oa=N.SCORER_OBSERVED_ATTENTION,
              nca=N.SCORER_NON_CAUSAL_ATTENTION, lagkv=N.SCORER_LAGKV, cur=N.SCORER_CUR, merging=N.SCORER_MERGING)


# --------------------------------------------------------------------------------------------------
# guarded arenas
# --------------------------------------------------------------------------------------------------
class Arena:
    """One allocation [guard | `offset` bytes | buffer of `nbytes` | guard]; the guards and the offset hold PATTERN."""

    def __init__(self, nbytes: int, offset: int = 0):
        self.start, self.n = GUARD + offset, nbytes
        self.raw = torch.full((2 * GUARD + offset + nbytes,), PATTERN, dtype=torch.uint8, device=DEV)
        self.buf = self.raw[self.start:self.start + nbytes]

    def fill(self, how: str, seed: int = 0):
        if how == "random":
            g = torch.Generator(device=DEV).manual_seed(seed)
            self.buf.copy_(torch.randint(0, 256, (self.n,), generator=g, device=DEV, dtype=torch.uint8))
        else:
            self.buf.fill_(0 if how == "zeros" else 0xFF)
        return self

    def view(self, dtype, shape):
        return self.buf.view(dtype).view(shape)

    def guards_intact(self) -> bool:
        return bool((self.raw[:self.start] == PATTERN).all() and (self.raw[self.start + self.n:] == PATTERN).all())


def out_arena(spec):
    if spec is None:
        return None
    dtype, shape = spec
    numel = 1
    for s in shape:
        numel *= s
    return Arena(numel * torch.empty((), dtype=dtype).element_size())


# --------------------------------------------------------------------------------------------------
# the calls
# --------------------------------------------------------------------------------------------------
@dataclass
class Case:
    name: str  # the C entry point
    p: object  # its kvp_problem
    args: tuple  # its arguments between the problem and the outputs
    outs: tuple  # per output slot: (dtype, shape), or None for a null output
    scorer: Optional[int]  # the workspace it takes (None: none)
    public: Callable[[], tuple]  # the same call through its native.* wrapper: the outputs in slot order
    flag: bool = True  # the call clears the workspace's leading region: kvp_workspace_check reads its flag
    keep: tuple = ()  # buffers that back addresses in `args`


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _kv(B, H, S, D, dtype, seed):
    g = _gen(seed)
    return (torch.randn(B, H, S, D, generator=g, device=DEV).to(dtype),
            torch.randn(B, H, S, D, generator=g, device=DEV).to(dtype))


def _scores(B, H, S, dtype, seed):
    return torch.randn(B, H, S, generator=_gen(seed + 7), device=DEV).to(dtype)


def _compress_outs(k, n_kept, scores=True):
    B, H, S, D = k.shape
    return ((k.dtype, (B, H, n_kept, D)), (k.dtype, (B, H, n_kept, D)), (torch.int32, (B, H, n_kept)),
            *(((k.dtype, (B, H, S)) if scores else None,) if scores is not None else ()))


def knorm(B, H, S, D, n_kept, dtype=torch.bfloat16, score=False):
    def make(seed):
        nat = _native()
        k, v = _kv(B, H, S, D, dtype, seed)
        if score:
            return Case("kvp_knorm_score", nat.make_problem(k, k, 0), (k,), ((dtype, (B, H, S)),), None,
                        lambda: (nat.knorm_score(k),))
        p = nat.make_problem(k, v, n_kept)
        return Case("kvp_knorm_compress", p, (k, v), _compress_outs(k, n_kept), SCORER["knorm"],
                    lambda: nat.knorm_compress(k, v, n_kept, True, True),
                    flag=nat.launches_per_compress(p, SCORER["knorm"]) > 1)
    return make


def keydiff(B, H, S, D, n_kept, dtype=torch.bfloat16, score=False):
    def make(seed):
        nat = _native()
        k, v = _kv(B, H, S, D, dtype, seed)
        if score:
            return Case("kvp_keydiff_score", nat.make_problem(k, k, 0), (k,), ((dtype, (B, H, S)),), SCORER["keydiff"],
                        lambda: (nat.keydiff_score(k),), flag=False)
        return Case("kvp_keydiff_compress", nat.make_problem(k, v, n_kept), (k, v), _compress_outs(k, n_kept),
                    SCORER["keydiff"], lambda: nat.keydiff_compress(k, v, n_kept, True, True))
    return make


def streaming(B, H, S, D, n_kept, n_sink=4, dtype=torch.float16, score=False):
    def make(seed):
        nat = _native()
        k, v = _kv(B, H, S, D, dtype, seed)
        if score:
            return Case("kvp_streaming_score", nat.make_problem(k, k, n_kept), (n_sink,), ((dtype, (B, H, S)),), None,
                        lambda: (nat.streaming_score(k, n_kept, n_sink),))
        return Case("kvp_streaming_compress", nat.make_problem(k, v, n_kept), (n_sink, k, v),
                    _compress_outs(k, n_kept, None), None,
                    lambda: nat.streaming_compress(k, v, n_kept, n_sink, return_indices=True))
    return make


def snapkv(B, H, G, S, D, w, n_kept, dtype=torch.bfloat16, score=False):
    def make(seed):
        nat = _native()
        k, v, q = snap_inputs(B, H, G, S, D, w, dtype, seed)
        if score:
            return Case("kvp_snapkv_score", nat.make_problem(k, k, 0, H * G), (k, q, w, 5), ((dtype, (B, H, S)),),
                        SCORER["snapkv"], lambda: (nat.snapkv_score(k, q, w, 5),))
        return Case("kvp_snapkv_compress", nat.make_problem(k, v, n_kept, H * G), (k, v, q, w, 5),
                    _compress_outs(k, n_kept), SCORER["snapkv"],
                    lambda: nat.snapkv_compress(k, v, q, w, 5, n_kept, True, True))
    return make


def ea(B, H, G, S, D, n_kept, cov=True, vnorm=True, dtype=torch.bfloat16, score=False):
    def make(seed):
        nat = _native()
        k, v, mu, c = ea_inputs(B, H, G, S, D, dtype, seed, cov=cov)
        a = (k, v, mu, c, 0.01, 4, int(vnorm))
        if score:
            return Case("kvp_expected_attention_score", nat.make_problem(k, v, 0, H * G), a, ((dtype, (B, H, S)),),
                        SCORER["ea"], lambda: (nat.expected_attention_score(*a[:4], 0.01, 4, vnorm),))
        return Case("kvp_expected_attention_compress", nat.make_problem(k, v, n_kept, H * G), a,
                    _compress_outs(k, n_kept), SCORER["ea"],
                    lambda: nat.expected_attention_compress(*a[:4], 0.01, 4, vnorm, n_kept, True, True))
    return make


def generic(B, H, S, D, n_kept, kind, dtype=torch.bfloat16):
    def make(seed):
        nat = _native()
        k, v = _kv(B, H, S, D, dtype, seed)
        sc, sst = nat._unit_stride_scores(_scores(B, H, S, dtype, seed))
        if kind == "select":
            p = nat.KvpProblem()
            p.B, p.Hkv, p.Hq, p.S, p.D, p.n_kept, p.dtype = B, H, H, S, 8, n_kept, nat._DTYPES[dtype]
            return Case("kvp_scores_select", p, (sc, sst), ((torch.int32, (B, H, n_kept)),), SCORER["generic"],
                        lambda: (nat.scores_select(sc, n_kept),))
        p = nat.make_problem(k, v, n_kept)
        if kind == "rerotate":
            inv = rope_inv_freq("theta500000", D).to(DEV)
            return Case("kvp_scores_compress_rerotate", p, (sc, sst, k, v, inv), _compress_outs(k, n_kept, None),
                        SCORER["generic"], lambda: nat.scores_compress_rerotate(sc, k, v, n_kept, inv, True))
        return Case("kvp_scores_compress", p, (sc, sst, k, v), _compress_outs(k, n_kept, None), SCORER["generic"],
                    lambda: nat.scores_compress(sc, k, v, n_kept, True))
    return make


def criticalkv(B, H, G, S, D, n_kept, n_first, dtype=torch.bfloat16, score=False, scores_out=True):
    def make(seed):
        nat = _native()
        v, wo, base = ckv_inputs(B, H, G, S, D, 256, dtype, seed)
        k = _kv(B, H, S, D, dtype, seed + 1)[0]
        bs, sst = nat._unit_stride_scores(base)
        w = (wo, wo.shape[0], int(wo.stride(0)), 1e-3, n_first)
        if score:
            return Case("kvp_criticalkv_score", nat.make_problem(v, v, 0, H * G), (v, bs, sst, *w),
                        ((dtype, (B, H, S)),), SCORER["ckv"], lambda: (nat.criticalkv_score(base, v, wo, 1e-3, n_first),),
                        flag=n_first > 0)
        return Case("kvp_criticalkv_compress", nat.make_problem(k, v, n_kept, H * G), (k, v, bs, sst, *w),
                    _compress_outs(k, n_kept, scores_out), SCORER["ckv"],
                    lambda: nat.criticalkv_compress(base, k, v, wo, 1e-3, n_first, n_kept, True, scores_out))
    return make


def observed(B, H, G, S, D, n_q, n_kept, dtype=torch.bfloat16, score=False):
    def make(seed):
        nat = _native()
        k, v, q = oa_inputs(B, H, G, S, n_q, D, dtype, seed)
        if score:
            return Case("kvp_observed_attention_score", nat.make_problem(k, k, 0, H * G), (k, q, n_q, 0.125),
                        ((dtype, (B, H, S)),), SCORER["oa"], lambda: (nat.observed_attention_score(k, q, 0.125),))
        return Case("kvp_observed_attention_compress", nat.make_problem(k, v, n_kept, H * G), (k, v, q, n_q, 0.125),
                    _compress_outs(k, n_kept), SCORER["oa"],
                    lambda: nat.observed_attention_compress(k, v, q, 0.125, n_kept, True, True))
    return make


def nca(B, H, G, S, D, cs, n_kept, dtype=torch.bfloat16, score=False):
    def make(seed):
        nat = _native()
        k, v, q = nca_inputs(B, H, G, S, D, dtype, seed)
        if score:
            return Case("kvp_non_causal_attention_score", nat.make_problem(k, v, 0, H * G), (k, v, q, cs),
                        ((dtype, (B, H, S)),), SCORER["nca"], lambda: (nat.non_causal_attention_score(k, v, q, cs),))
        return Case("kvp_non_causal_attention_compress", nat.make_problem(k, v, n_kept, H * G), (k, v, q, cs),
                    _compress_outs(k, n_kept), SCORER["nca"],
                    lambda: nat.non_causal_attention_compress(k, v, q, cs, n_kept, True, True))
    return make


def lagkv(B, H, S, D, lag, cross, n_kept, dtype=torch.bfloat16, score=False):
    def make(seed):
        nat = _native()
        k, v = lagkv_inputs(B, H, S, D, dtype, seed)
        a = (k, v, 4, lag, int(cross))
        if score:
            return Case("kvp_lagkv_score", nat.make_problem(k, v, 0), a, ((dtype, (B, H, S)),), SCORER["lagkv"],
                        lambda: (nat.lagkv_score(k, v, 4, lag, cross),), flag=False)
        return Case("kvp_lagkv_compress", nat.make_problem(k, v, n_kept), a, _compress_outs(k, n_kept),
                    SCORER["lagkv"], lambda: nat.lagkv_compress(k, v, 4, lag, cross, n_kept, True, True))
    return make


def cur(B, H, S, D, window, r, n_kept, dtype=torch.float16, score=False):
    def make(seed):
        nat = _native()
        k, v = _kv(B, H, S, D, dtype, seed)
        G = torch.randn(D, r, generator=_gen(seed + 3), device=DEV) / r ** 0.5 if r else None
        a = nat._cur_inputs(k, v, 2, "kv_avg", window, G)
        if score:
            return Case("kvp_cur_score", nat.make_problem(k, v, 0), a, ((dtype, (B, H, S)),), SCORER["cur"],
                        lambda: (nat.cur_score(k, v, 2, "kv_avg", window, G),))
        return Case("kvp_cur_compress", nat.make_problem(k, v, n_kept), a, _compress_outs(k, n_kept), SCORER["cur"],
                    lambda: nat.cur_compress(k, v, 2, "kv_avg", window, G, n_kept, True, True))
    return make


def merging(B, H, S, D, n_kept, frac=0.5, dtype=torch.bfloat16, merge=False):
    def make(seed):
        nat = _native()
        k, v = _kv(B, H, S, D, dtype, seed)
        plan = ((torch.int32, (B, H, S - n_kept)), (torch.float32, (B, H, S - n_kept)))
        if merge:
            g = _gen(seed + 5)
            rows = [torch.randperm(S, generator=g, device=DEV)[:n_kept].sort().values for _ in range(B * H)]
            kept = torch.cat(rows).to(torch.int32).view(B, H, n_kept)
            # an empty tensor's address is null: n_kept == 0 gets the address of a live buffer instead
            live = torch.zeros(4, dtype=torch.int32, device=DEV)
            arg = kept if n_kept else live.data_ptr()
            return Case("kvp_merging_merge", nat.make_problem(k, v, n_kept), (k, v, arg, 0.1, frac),
                        ((dtype, (B, H, n_kept, D)), *plan), SCORER["merging"],
                        lambda: nat.merging_merge(k, v, kept, 0.1, frac, True), flag=False, keep=(live,))
        sc, sst = nat._unit_stride_scores(_scores(B, H, S, dtype, seed))
        return Case("kvp_merging_compress", nat.make_problem(k, v, n_kept), (sc, sst, k, v, 0.1, frac),
                    (*_compress_outs(k, n_kept, None), *plan), SCORER["merging"],
                    lambda: nat.merging_compress(sc, k, v, 0.1, frac, n_kept, True, True))
    return make


# id -> case builder (seed -> Case). The shapes aim at the tails: S = 1, S off every multiple of 64 / 128 / 256 (1000,
# 4097), S = 512, odd row counts B * Hkv (3 x 1, 1 x 5), every head_dim class, n_kept = 1, odd, S - 1 and S.
CASES = {
    "knorm_cluster": knorm(1, 8, 5888, 128, 2945),
    "knorm_fused": knorm(1, 8, 5889, 128, 1, dtype=torch.float16),
    "knorm_odd_rows": knorm(3, 1, 1000, 72, 999),
    "knorm_s1": knorm(1, 5, 1, 256, 1),
    "knorm_two_kernels": knorm(1, 1, 131073, 128, 131072),
    "knorm_score": knorm(1, 5, 4097, 256, 0, score=True),
    "keydiff_score": keydiff(3, 1, 1000, 8, 0, score=True),
    "keydiff_compress": keydiff(1, 5, 4097, 256, 2049),
    "keydiff_compress_s1": keydiff(1, 5, 1, 72, 1, dtype=torch.float16),
    "streaming_score": streaming(1, 5, 1000, 64, 501, score=True),
    "streaming_compress": streaming(3, 1, 4097, 8, 999),
    "snapkv_score_g1_w257": snapkv(1, 1, 1, 1000, 128, 257, 0, score=True),
    "snapkv_compress_g1_w257": snapkv(3, 1, 1, 1000, 128, 257, 999),
    "snapkv_compress_g1_w384": snapkv(1, 5, 1, 4097, 64, 384, 1, dtype=torch.float16),
    "snapkv_compress_g1_w511": snapkv(1, 2, 1, 512, 128, 511, 511),
    "snapkv_score_g4": snapkv(1, 2, 4, 4097, 64, 64, 0, score=True),
    "snapkv_compress_g4": snapkv(3, 1, 4, 512, 128, 100, 257),
    "ea_score_cov_vnorm": ea(1, 2, 4, 1000, 128, 0, score=True),
    "ea_compress_cov_vnorm": ea(1, 5, 2, 4097, 64, 2049),
    "ea_compress_plain": ea(3, 1, 4, 1000, 128, 1, cov=False, vnorm=False, dtype=torch.float16),
    "ea_score_cov": ea(3, 1, 2, 512, 64, 0, vnorm=False, score=True),
    "ea_compress_vnorm": ea(1, 2, 1, 1000, 64, 999, cov=False),
    "scores_compress": generic(1, 5, 1000, 72, 501, "compress"),
    "scores_compress_s1": generic(1, 5, 1, 256, 1, "compress", dtype=torch.float16),
    "scores_select": generic(3, 1, 4097, 8, 4096, "select"),
    "scores_select_s1": generic(1, 5, 1, 8, 1, "select"),
    "rerotate": generic(3, 1, 1000, 64, 501, "rerotate"),
    "rerotate_all": generic(1, 5, 512, 128, 512, "rerotate", dtype=torch.float16),
    "ckv_score": criticalkv(1, 2, 4, 1000, 128, 0, 0, score=True),
    "ckv_score_first": criticalkv(3, 1, 2, 4097, 64, 0, 100, score=True),
    "ckv_compress": criticalkv(1, 5, 1, 1000, 64, 1, 0),
    "ckv_compress_first": criticalkv(3, 1, 2, 512, 128, 257, 100),
    "ckv_compress_first_null_scores": criticalkv(1, 2, 4, 1000, 128, 501, 501, scores_out=False),
    "oa_score_lt": observed(1, 2, 2, 1000, 128, 100, 0, score=True),
    "oa_compress_lt": observed(3, 1, 4, 4097, 64, 33, 2049, dtype=torch.float16),
    "oa_score_eq": observed(1, 5, 1, 257, 64, 257, 0, score=True),
    "oa_compress_eq": observed(1, 2, 2, 512, 128, 512, 511),
    "nca_score_256": nca(1, 2, 2, 1000, 128, 256, 0, score=True),
    "nca_compress_256": nca(3, 1, 1, 4097, 64, 256, 1),
    "nca_compress_128": nca(1, 5, 4, 1000, 64, 128, 501),
    "nca_score_128": nca(1, 2, 8, 512, 128, 128, 0, score=True, dtype=torch.float16),
    "lagkv_score": lagkv(1, 5, 1000, 72, 64, False, 0, score=True),
    "lagkv_score_cross": lagkv(3, 1, 4097, 256, 128, True, 0, score=True),
    "lagkv_compress": lagkv(3, 1, 1000, 128, 100, False, 501),
    "lagkv_compress_cross": lagkv(1, 5, 4097, 8, 1024, True, 4096, dtype=torch.float16),
    "lagkv_compress_s1": lagkv(1, 5, 1, 64, 1, True, 1),
    "cur_score_proj": cur(1, 5, 1000, 72, 16, 8, 0, score=True),
    "cur_score_plain": cur(3, 1, 4097, 256, 0, 0, 0, score=True),
    "cur_compress_proj": cur(3, 1, 4097, 128, 1024, 32, 2049),
    "cur_compress_plain": cur(1, 5, 1000, 8, 0, 0, 999, dtype=torch.bfloat16),
    "cur_compress_s1": cur(1, 5, 1, 64, 1, 4, 1),
    "merging_compress": merging(1, 2, 1000, 128, 501),
    "merging_compress_all_kept": merging(3, 1, 257, 64, 257),
    "merging_compress_one_kept": merging(1, 5, 512, 72, 1, frac=1.0, dtype=torch.float16),
    "merging_merge": merging(1, 5, 1000, 64, 333, merge=True),
    "merging_merge_odd": merging(3, 1, 4097, 256, 4096, frac=1.0, merge=True),
}
# compress / select / merge calls with n_kept == 0
EMPTY = {
    "knorm": knorm(1, 5, 1000, 128, 0),
    "keydiff": keydiff(3, 1, 1000, 64, 0),
    "snapkv": snapkv(1, 1, 1, 1000, 128, 300, 0),
    "ea": ea(1, 2, 4, 1000, 128, 0),
    "scores_select": generic(3, 1, 1000, 8, 0, "select"),
    "scores_compress": generic(3, 1, 1000, 64, 0, "compress"),
    "rerotate": generic(3, 1, 1000, 64, 0, "rerotate"),
    "ckv": criticalkv(1, 2, 4, 1000, 128, 0, 0),
    "oa": observed(1, 2, 2, 1000, 128, 100, 0),
    "nca": nca(1, 2, 2, 1000, 128, 256, 0),
    "lagkv": lagkv(1, 5, 1000, 72, 64, False, 0),
    "cur": cur(1, 5, 1000, 72, 16, 8, 0),
    "merging_compress": merging(1, 2, 1000, 128, 0),
    "merging_merge": merging(1, 2, 1000, 128, 0, merge=True),
}

_TLS = threading.local()  # the workspace the replaced native._workspace hands out on this thread


@pytest.fixture
def private_workspace(monkeypatch):
    monkeypatch.setattr(_native(), "_workspace", lambda p, scorer, device: _TLS.ws)


def _ws_arena(case: Case, offset: int = 0) -> Optional[Arena]:
    return None if case.scorer is None else Arena(_native().workspace_bytes(case.p, case.scorer), offset)


def enqueue(case: Case, ws: Optional[torch.Tensor], outs: list):
    """The call of `case` on the current stream: its workspace the bytes `ws`, its outputs the views of `outs`."""
    _TLS.ws = ws
    views = [None if a is None else a.view(*spec) for a, spec in zip(outs, case.outs)]
    # an empty output's tensor address is null: it gets its arena's address, as a caller's empty buffer would
    ptrs = [a.raw.data_ptr() + a.start if v is not None and v.numel() == 0 else v for a, v in zip(outs, views)]
    _native()._enqueue(case.name, torch.device(DEV), case.p, *case.args, *ptrs, scorer=case.scorer)
    return views


def _inputs(case: Case) -> list:
    return [a for a in case.args if isinstance(a, torch.Tensor)]


def _bits(t: Optional[torch.Tensor]):
    return None if t is None else t.contiguous().view(torch.uint8).clone()


def same(a, b) -> bool:
    if a is None or b is None:
        return a is None and b is None
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(_bits(a), _bits(b))


def run_alone(case: Case, ws_fill: str, out_fill: str, seed: int = 0, offset: int = 0) -> list:
    """One call on a fresh arena per buffer, with bars 2-4 checked; returns copies of the outputs."""
    nat = _native()
    ws = _ws_arena(case, offset)
    if ws is not None:
        ws.fill(ws_fill, seed)
    outs = [out_arena(s) for s in case.outs]
    for a in outs:
        if a is not None:
            a.fill(out_fill)
    before = [_bits(t) for t in _inputs(case)]
    views = enqueue(case, None if ws is None else ws.buf, outs)
    torch.cuda.synchronize()
    what = f"{case.name} ws={ws_fill} out={out_fill} offset={offset}"
    assert ws is None or ws.guards_intact(), f"{what}: a workspace guard byte changed"
    bad = [i for i, a in enumerate(outs) if a is not None and not a.guards_intact()]
    assert not bad, f"{what}: a guard byte of output slot(s) {bad} changed"
    if ws is not None and case.flag:
        nat.workspace_check(case.p, case.scorer, ws.buf)
    assert all(torch.equal(b, _bits(t)) for b, t in zip(before, _inputs(case))), f"{what}: an input changed"
    return [None if v is None else v.clone() for v in views]


def assert_same_outputs(got: list, want: list, what: str):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert same(g, w), f"{what}: output slot {i} differs"


@gpu
@pytest.mark.parametrize("cid", list(CASES))
def test_outputs_do_not_depend_on_workspace_or_output_contents(cid, private_workspace):
    case = CASES[cid](100 + len(cid))
    nat = _native()
    want_path = {"knorm_cluster": 1, "knorm_fused": 2, "knorm_two_kernels": 3}.get(cid)
    if want_path is not None:
        assert nat.launches_per_compress(case.p, SCORER["knorm"]) == want_path, f"{cid}: not the intended path"
    ref = None
    for wf in WS_FILLS:
        for of in OUT_FILLS:
            got = run_alone(case, wf, of, seed=len(cid))
            if ref is None:
                ref = got
            assert_same_outputs(got, ref, f"{cid}: ws={wf} out={of} against ws={WS_FILLS[0]} out={OUT_FILLS[0]}")
    public = case.public()
    torch.cuda.synchronize()
    assert_same_outputs(list(public)[:len(case.outs)], ref, f"{cid}: the public wrapper")


@gpu
@pytest.mark.parametrize("cid", list(EMPTY))
def test_n_kept_zero_touches_nothing(cid, private_workspace):
    case = EMPTY[cid](7)
    ws = _ws_arena(case)
    outs = [out_arena(s) for s in case.outs]
    arenas = [a for a in (ws, *outs) if a is not None]
    for i, a in enumerate(arenas):
        a.fill("random", seed=i)
    before = [a.raw.clone() for a in arenas]
    enqueue(case, None if ws is None else ws.buf, outs)
    torch.cuda.synchronize()
    assert all(torch.equal(b, a.raw) for b, a in zip(before, arenas)), f"{cid}: an n_kept == 0 call wrote memory"


# the same scorer and shape twice in a row on new inputs, then shapes that grow and shrink
SEQUENCE = [("ea_compress_cov_vnorm", 1), ("snapkv_compress_g1_w257", 1), ("snapkv_compress_g1_w257", 2),
            ("keydiff_compress", 1), ("cur_compress_proj", 1), ("cur_compress_proj", 2), ("knorm_fused", 1),
            ("oa_compress_lt", 1), ("oa_compress_lt", 2), ("nca_compress_256", 1), ("lagkv_compress_cross", 1),
            ("ckv_compress_first", 1), ("ckv_compress_first", 2), ("merging_compress", 1), ("merging_compress", 2),
            ("scores_select", 1), ("rerotate", 1), ("ea_compress_plain", 1), ("ea_compress_plain", 2),
            ("snapkv_compress_g4", 1), ("keydiff_score", 1), ("keydiff_score", 2), ("lagkv_score", 1),
            ("merging_merge", 1), ("merging_merge", 2), ("nca_compress_128", 1), ("knorm_two_kernels", 1)]


@gpu
def test_shared_workspace_sequence_matches_each_call_alone(private_workspace):
    nat = _native()
    cases = [CASES[cid](1000 * seed + i) for i, (cid, seed) in enumerate(SEQUENCE)]
    alone = [run_alone(c, "ones", "zeros") for c in cases]
    shared = Arena(max(nat.workspace_bytes(c.p, c.scorer) for c in cases)).fill("random", seed=3)
    for i, ((cid, seed), c) in enumerate(zip(SEQUENCE, cases)):
        # the head of the shared buffer, exactly as large as the call asks for
        got = enqueue(c, shared.buf[:nat.workspace_bytes(c.p, c.scorer)], [out_arena(s) for s in c.outs])
        torch.cuda.synchronize()
        assert shared.guards_intact(), f"call {i} ({cid}): a guard of the shared workspace changed"
        assert_same_outputs(got, alone[i], f"call {i} ({cid}, seed {seed}) on the shared workspace")


STREAM_A = [("ea_compress_cov_vnorm", 1), ("cur_compress_proj", 1), ("ea_score_cov_vnorm", 2), ("cur_score_proj", 1)]
STREAM_B = [("snapkv_compress_g1_w384", 1), ("keydiff_compress", 1), ("merging_compress", 1), ("snapkv_score_g4", 1),
            ("merging_merge", 1)]


def _serial(lists):
    cases = [[CASES[cid](50 * seed + 7 * i) for i, (cid, seed) in enumerate(lst)] for lst in lists]
    return cases, [[run_alone(c, "ones", "zeros") for c in cs] for cs in cases]


def _own_workspace(cases) -> Arena:
    nat = _native()
    return Arena(max(nat.workspace_bytes(c.p, c.scorer) for c in cases)).fill("random", seed=9)


def _run_list(cases, arena: Arena) -> list:
    res = []
    for c in cases:
        ws = arena.buf[:_native().workspace_bytes(c.p, c.scorer)]
        res.append(enqueue(c, ws, [out_arena(s) for s in c.outs]))
    return res


@gpu
def test_two_streams_interleaved_match_serial(private_workspace):
    (ca, cb), (ra, rb) = _serial([STREAM_A, STREAM_B])
    wa, wb = _own_workspace(ca), _own_workspace(cb)
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    for s in (sa, sb):
        s.wait_stream(torch.cuda.current_stream())
    got_a, got_b = [], []
    for i in range(max(len(ca), len(cb))):
        if i < len(ca):
            with torch.cuda.stream(sa):
                got_a += _run_list([ca[i]], wa)
        if i < len(cb):
            with torch.cuda.stream(sb):
                got_b += _run_list([cb[i]], wb)
    torch.cuda.synchronize()
    assert wa.guards_intact() and wb.guards_intact()
    for got, want, lst in ((got_a, ra, STREAM_A), (got_b, rb, STREAM_B)):
        for g, w, (cid, _) in zip(got, want, lst):
            assert_same_outputs(g, w, f"{cid} on its own stream")


@gpu
def test_two_host_threads_match_serial(private_workspace):
    (ca, cb), (ra, rb) = _serial([STREAM_A, STREAM_B])
    wa, wb = _own_workspace(ca), _own_workspace(cb)
    results, errors = {}, []
    torch.cuda.synchronize()

    def worker(key, cases, arena):
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                results[key] = _run_list(cases, arena)
            s.synchronize()
        except Exception as e:  # reported by the main thread
            errors.append(e)

    threads = [threading.Thread(target=worker, args=("a", ca, wa)), threading.Thread(target=worker, args=("b", cb, wb))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    torch.cuda.synchronize()
    for key, want, lst in (("a", ra, STREAM_A), ("b", rb, STREAM_B)):
        for g, w, (cid, _) in zip(results[key], want, lst):
            assert_same_outputs(g, w, f"{cid} on thread {key}")


# one call per scorer on a workspace whose base is 16 mod 256 bytes. No scratch access is wider than 16 bytes, and the
# one TMA map on scratch (Merging's gathered keys) needs a 16-byte aligned address.
ALIGNMENT = ["knorm_fused", "keydiff_compress", "snapkv_compress_g1_w257", "ea_compress_cov_vnorm", "rerotate",
             "scores_select", "ckv_compress_first", "oa_compress_lt", "nca_compress_128", "lagkv_compress_cross",
             "cur_compress_proj", "merging_compress", "merging_merge"]


@gpu
@pytest.mark.parametrize("cid", ALIGNMENT)
def test_workspace_base_16_mod_256(cid, private_workspace):
    case = CASES[cid](31)
    want = run_alone(case, "ones", "zeros")
    got = run_alone(case, "random", "ones", seed=5, offset=16)
    assert_same_outputs(got, want, f"{cid}: workspace at 16 mod 256")
