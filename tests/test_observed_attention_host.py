"""ObservedAttention on the GPU-less box: the C ABI's checks of the two new entry points, the argument lists of their
wrappers, the schedule of the two tensor-core passes, and the press against the UNMODIFIED reference through the
oracle-backed stand-ins.

Statuses: every argument of kvp_observed_attention_score / kvp_observed_attention_compress made invalid on its own (or set
to another valid value), and every pair of such changes to two different arguments, against a restatement of the
documented check order (include/kvpress_b200.h). The pointers are fake, 16-byte aligned or not, and never dereferenced:
the calls run in a child process that sees no GPU, so a call that passes every check fails at its first CUDA call with
KVP_ERR_CUDA (-6).

Reference: what the reference's ObservedAttentionPress computes (eager attention) on the seeded tiny models is stored in
tests/golden/observed_attention_reference.npz. To re-record it from a checkout of the reference (located as in
oracle/build_ref.py):  KVP_RECORD_OBSERVED_ATTENTION=1 python -m pytest tests/test_observed_attention_host.py
"""
import ctypes
import itertools
import json
import math
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
from transformers import DynamicCache

from kvpress_b200 import DecodingPress, ObservedAttentionPress, native
from tests import cpu_backend, observed_attention_backend
from tests.test_native_marshalling import _kv, rec  # noqa: F401  (fixture)
from tests.test_reference_differential import _import_reference, _rows_signature, close
from tests.tiny_models import tiny_llama, tiny_qwen3

ROOT = Path(__file__).resolve().parent.parent
STORE = ROOT / "tests" / "golden" / "observed_attention_reference.npz"
RECORD = os.environ.get("KVP_RECORD_OBSERVED_ATTENTION") == "1"

# --------------------------------------------------------------------------------------------------
# C ABI statuses
# --------------------------------------------------------------------------------------------------
GOOD, ODD16 = 0x10000, 0x1000C  # aligned; 4-byte but not 16-byte aligned
FIELDS = dict(B=1, Hkv=2, Hq=4, S=1000, D=128, n_kept=500, dtype=0)
STRIDES = (256000, 128000, 128)
VALID = dict(K=GOOD, V=GOOD, q=GOOD, n_q=1000, scaling=0.125, K_out=GOOD, V_out=GOOD, idx=GOOD, scores=GOOD, ws=GOOD,
             ws_bytes="enough", stream=0)
SLOTS = {
    "kvp_observed_attention_score": "K q n_q scaling scores ws ws_bytes stream",
    "kvp_observed_attention_compress": "K V q n_q scaling K_out V_out idx scores ws ws_bytes stream",
}
CHANGES = {  # slot -> {label: value}
    "p": {"null": None},
    "dtype": {"3": 3},
    "S": {"0": 0},
    "D": {"12": 12, "64": 64},
    "Hq": {"5": 5},
    "n_kept": {"-1": -1, "0": 0, "1000": 1000},
    "k_stride": {"s100": (256000, 128000, 100)},
    "K": {"null": None, "odd": ODD16},
    "V": {"null": None, "odd": ODD16},
    "q": {"null": None, "odd": ODD16},
    "n_q": {"0": 0, "-1": -1, "1": 1, "999": 999, "1001": 1001},
    "scaling": {"0": 0.0, "-1": -1.0, "inf": math.inf, "nan": math.nan, "1": 1.0},
    "K_out": {"null": None},
    "V_out": {"null": None, "odd": ODD16},
    "idx": {"null": None},
    "scores": {"null": None},
    "ws": {"null": None, "odd": ODD16},
    "ws_bytes": {"short": "short"},
}
PROBLEM = ("dtype", "S", "D", "Hq", "n_kept", "k_stride")


def _align256(n: int) -> int:
    return (n + 255) // 256 * 256


def expected(name: str, c: dict) -> int:
    """The documented check order: validate -> n_kept == 0 short cut (compress) -> K / V / outputs (compress) ->
    null / alignment of q (and K, scores for the score call) -> n_q -> scaling -> workspace."""
    f = {**FIELDS, **{k: v for k, v in c.items() if k in FIELDS}}
    a = {**VALID, **{k: v for k, v in c.items() if k not in FIELDS}}
    compress = name.endswith("compress")
    if c.get("p", 0) is None:
        return -1
    if f["dtype"] not in (0, 1):
        return -3
    if f["S"] <= 0 or f["D"] % 8 or f["Hq"] % FIELDS["Hkv"]:
        return -2
    if not 0 <= f["n_kept"] <= f["S"]:
        return -7
    if "k_stride" in c:
        return -4
    if compress:
        if f["n_kept"] == 0:
            return 0
        io = [a["K"], a["V"], a["K_out"], a["V_out"]]
        if None in io:
            return -1
        if any(x % 16 for x in io):
            return -4
        nulls, aligned = [a["q"]], [a["q"]]
    else:
        nulls, aligned = [a["K"], a["q"], a["scores"]], [a["K"], a["q"]]
    if None in nulls:
        return -1
    if any(x % 16 for x in aligned):
        return -4
    if not 1 <= a["n_q"] <= f["S"]:
        return -7
    if not (math.isfinite(a["scaling"]) and a["scaling"] > 0):
        return -7
    if a["ws"] is None:
        return -1
    if a["ws"] % 16:
        return -4
    if a["ws_bytes"] == "short":
        # one byte short of the size for n_q = S; the per-row normalisers of fewer rows may still fit
        qrows = lambda n: _align256(4 * f["B"] * f["Hq"] * n)  # noqa: E731
        return -5 if qrows(a["n_q"]) == qrows(f["S"]) else -6
    return -6


def _cases(name: str) -> dict:
    slots = ["p", *PROBLEM, *SLOTS[name].split()]
    singles = [(s, label, v) for s in slots for label, v in CHANGES.get(s, {}).items()]
    cases = {"valid": {}, **{f"{s}={label}": {s: v} for s, label, v in singles}}
    cases.update({f"{s1}={l1},{s2}={l2}": {s1: v1, s2: v2}
                  for (s1, l1, v1), (s2, l2, v2) in itertools.combinations(singles, 2) if s1 != s2})
    return cases


def statuses() -> dict:
    """Every case's status. Run only in a process that sees no GPU."""
    import importlib.util

    assert torch.cuda.device_count() == 0, "the status cases pass fake device pointers: they must not see a GPU"
    spec = importlib.util.spec_from_file_location("kvp_native", ROOT / "kvpress_b200" / "native.py")
    nat = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(nat)
    lib = nat.load()

    def problem(c):
        p = nat.KvpProblem()
        for k, v in {**FIELDS, **{k: v for k, v in c.items() if k in FIELDS}}.items():
            setattr(p, k, v)
        p.k_stride = (ctypes.c_int64 * 3)(*c.get("k_stride", STRIDES))
        p.v_stride = (ctypes.c_int64 * 3)(*STRIDES)
        return p

    need = ctypes.c_size_t(0)
    assert lib.kvp_workspace_bytes(ctypes.byref(problem({})), nat.SCORER_OBSERVED_ATTENTION, ctypes.byref(need)) == 0
    out = {}
    for name in SLOTS:
        for label, c in _cases(name).items():
            args = [None if c.get("p", 0) is None else ctypes.byref(problem(c))]
            for slot in SLOTS[name].split():
                v = c.get(slot, VALID[slot])
                if slot == "ws_bytes":
                    v = need.value - 1 if v == "short" else need.value
                elif slot == "idx" and v is not None:
                    v = ctypes.cast(ctypes.c_void_p(v), ctypes.POINTER(ctypes.c_int32))
                args.append(v)
            out[f"{name}({label})"] = getattr(lib, name)(*args)
    return out


def test_every_status_of_the_observed_attention_entry_points_follows_the_check_order():
    env = {k: v for k, v in os.environ.items() if not k.startswith("KVP_")}
    env["CUDA_VISIBLE_DEVICES"] = ""
    code = "import json, tests.test_observed_attention_host as m; print(json.dumps(m.statuses()))"
    r = subprocess.run([sys.executable, *(["-s"] if sys.flags.no_user_site else []), "-c", code], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    want = {f"{name}({label})": expected(name, c) for name in SLOTS for label, c in _cases(name).items()}
    assert sorted(got) == sorted(want) and len(got) > 900
    diffs = [f"{k}: {got[k]} != {want[k]}" for k in want if got[k] != want[k]]
    assert not diffs, f"{len(diffs)} differences, first ones:\n" + "\n".join(diffs[:30])


def test_workspace_and_launch_count_of_the_new_scorer_id():
    lib = native.load()
    p = native.KvpProblem()
    p.B, p.Hkv, p.Hq, p.D, p.n_kept, p.dtype = 1, 8, 32, 128, 0, 0
    prev = 0
    for S in (1, 2, 255, 256, 257, 4096, 16384, 131072):
        p.S = S
        obs, generic, n = ctypes.c_size_t(0), ctypes.c_size_t(0), ctypes.c_int(0)
        assert lib.kvp_workspace_bytes(ctypes.byref(p), native.SCORER_OBSERVED_ATTENTION, ctypes.byref(obs)) == 0
        assert lib.kvp_workspace_bytes(ctypes.byref(p), native.SCORER_GENERIC, ctypes.byref(generic)) == 0
        # the normaliser of every query row at n_q = S, and the fp32 column sums
        assert obs.value - generic.value >= 32 * S * 4 + 8 * S * 4
        assert obs.value >= prev
        prev = obs.value
        assert lib.kvp_launches_per_compress(ctypes.byref(p), native.SCORER_OBSERVED_ATTENTION, ctypes.byref(n)) == 0
        assert n.value == 5


# --------------------------------------------------------------------------------------------------
# wrappers: each argument after the kvp_problem, in order, down to the workspace and the stream
# --------------------------------------------------------------------------------------------------
def test_observed_attention_wrappers_pass_their_full_argument_list(rec, monkeypatch):  # noqa: F811
    workspaces = []
    real_workspace = native._workspace

    def spy(p, scorer, device):
        workspaces.append((scorer, real_workspace(p, scorer, device)))
        return workspaces[-1][1]

    monkeypatch.setattr(native, "_workspace", spy)
    P = lambda t: t.data_ptr()  # noqa: E731
    k, v = _kv(B=2, H=2, S=64, D=64)
    q = torch.randn(2, 8, 40, 64).to(torch.bfloat16)

    def last(name, n_kept):
        got, p, a = rec.calls[-1]
        assert got == name and (p["n_kept"], p["Hq"], p["D"], p["S"]) == (n_kept, 8, 64, 64)
        s, ws = workspaces[-1]
        problem = native.make_problem(k, v, n_kept, 8)
        assert s == native.SCORER_OBSERVED_ATTENTION
        assert a[-3:] == [ws.data_ptr(), native.workspace_bytes(problem, native.SCORER_OBSERVED_ATTENTION), 0]
        return a[:-3]

    sc = native.observed_attention_score(k, q, 0.25)
    a = last("kvp_observed_attention_score", 0)
    assert a == [P(k), P(q), 40, 0.25, P(sc)] and isinstance(a[3], float)
    k_out, v_out, idx, sc = native.observed_attention_compress(k, v, q, 0.5, 20, return_indices=True,
                                                               return_scores=True)
    assert last("kvp_observed_attention_compress", 20) == \
        [P(k), P(v), P(q), 40, 0.5, P(k_out), P(v_out), P(idx), P(sc)]
    qt = torch.randn(2, 40, 8, 64).to(torch.bfloat16).transpose(1, 2)  # a view: made contiguous
    native.observed_attention_compress(k, v, qt, 1, 20)
    a = last("kvp_observed_attention_compress", 20)
    assert a[2] != P(qt) and a[3:5] == [40, 1.0] and a[7:] == [0, 0]
    with pytest.raises(RuntimeError, match="n_q"):
        native.observed_attention_score(k, torch.randn(2, 8, 65, 64).to(torch.bfloat16), 0.25)
    with pytest.raises(RuntimeError, match="dtype"):
        native.observed_attention_score(k, q.half(), 0.25)


# --------------------------------------------------------------------------------------------------
# schedule of the two tensor-core passes, restated from csrc/observed_attention.cu (launch_obs_t)
# --------------------------------------------------------------------------------------------------
TILE = 128


def stats_items(R: int, S: int, n_q: int, G: int):
    """Pass 1: item u = (block qb = n_blocks - 1 - u // R, row u % R); work = K tiles up to the block's diagonal."""
    qpos = 128 if G == 1 else 64
    n_blocks = -(-n_q // qpos)
    u = np.arange(R * n_blocks)
    qb, row = n_blocks - 1 - u // R, u % R
    end = np.minimum(S, S - n_q + qb * qpos + qpos)
    return np.stack([qb, row], 1), -(-end // TILE)


def colsum_items(R: int, S: int, n_q: int, G: int):
    """Pass 2: item u = (key tile kt = u // R, row u % R); work = G x the 128-row Q chunks from the tile's diagonal."""
    n_kt = -(-S // TILE)
    u = np.arange(R * n_kt)
    kt, row = u // R, u % R
    i_min = np.maximum(0, kt * TILE - (S - n_q))
    return np.stack([kt, row], 1), G * (-(-(n_q - i_min) // TILE))


def deal(n_items: int, sm: int):
    """Persistent grid of min(SMs, items) CTAs; CTA p takes the items p, p + grid, ..."""
    grid = min(sm, n_items)
    return np.arange(n_items) % grid, grid


SHAPES = [(S, n_q) for S in (1, 2, 127, 128, 129, 255, 1000, 4097, 16384, 32768, 65600, 131072)
          for n_q in sorted({S, max(1, S - 1), min(S, 130), min(S, 7), 1})]


@pytest.mark.parametrize("sm", [1, 78, 132])
def test_observed_attention_partition_is_balanced_and_complete(sm):
    for (S, n_q), R, G in itertools.product(SHAPES, (1, 8, 32), (1, 3, 4, 8)):
        for name, (items, work) in (("stats", stats_items(R, S, n_q, G)), ("colsum", colsum_items(R, S, n_q, G))):
            what = f"{name} S={S} n_q={n_q} R={R} G={G} sm={sm}"
            # complete, no item twice: the (block or tile, row) pairs are exactly the grid of the pass
            n_major = -(-n_q // (128 if G == 1 else 64)) if name == "stats" else -(-S // TILE)
            assert len(items) == n_major * R and len({tuple(x) for x in items}) == len(items), what
            assert items[:, 0].min() == 0 and items[:, 0].max() == n_major - 1, what
            assert (work >= 1).all() and (np.diff(work) <= 0).all(), what  # dealt in non-increasing work
            cta, grid = deal(len(items), sm)
            load = np.bincount(cta, weights=work, minlength=grid)
            assert (load > 0).all(), what
            # balanced: no CTA holds more than the mean plus one item's work
            assert load.max() <= work.sum() / grid + work.max(), what


# --------------------------------------------------------------------------------------------------
# the press against the unmodified reference (CPU stand-ins)
# --------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ref():
    stored = {} if RECORD or not STORE.exists() else dict(np.load(STORE))
    recorded = {}

    def result(key: str, compute) -> dict:
        if RECORD:
            out = {k: np.asarray(x.detach().numpy() if torch.is_tensor(x) else x)
                   for k, x in compute(_import_reference()).items()}
            out = {k: x.astype(np.float32) if x.dtype == np.float64 else x.astype(np.int32) if x.dtype == np.int64
                   else x for k, x in out.items()}
            recorded.update({f"{key}|{k}": x for k, x in out.items()})
            return out
        out = {k.split("|", 1)[1]: x for k, x in stored.items() if k.split("|", 1)[0] == key}
        assert out, f"no stored reference result for {key}"
        return out

    yield result
    if RECORD:
        np.savez_compressed(STORE, **recorded)


def _ids(n=160, seed=5):
    g = torch.Generator().manual_seed(seed)
    return torch.stack([torch.randperm(250, generator=g)[:n] + 2 for _ in range(2)])


def _model(family, attn):
    m = tiny_llama() if family == "llama" else tiny_qwen3()
    m.config._attn_implementation = attn
    return m


def _signatures(cache) -> dict:
    return {"len": cache.get_seq_length(), **{f"sig{i}": _rows_signature(la.keys, la.values)
                                               for i, la in enumerate(cache.layers)}}


@pytest.mark.parametrize("ratio", [0.25, 0.5, 0.7])
@pytest.mark.parametrize("family", ["llama", "qwen3"])
def test_observed_attention_keeps_the_reference_rows(monkeypatch, ref, ratio, family):
    cpu_backend.install(monkeypatch)
    observed_attention_backend.install(monkeypatch)
    ids = _ids()

    def reference(kvpress):
        model, cache = _model(family, "eager"), DynamicCache()
        with kvpress.ObservedAttentionPress(compression_ratio=ratio)(model):
            model.model(input_ids=ids, past_key_values=cache, cache_position=torch.arange(ids.shape[1]))
        return _signatures(cache)

    want = ref(f"observed/{ratio}/{family}", reference)
    # same attention implementation as the reference, so that later layers see bit-equal hidden states; the press
    # ignores the eager weights it is handed
    model, ours = _model(family, "eager"), DynamicCache()
    with ObservedAttentionPress(compression_ratio=ratio)(model):
        model.model(input_ids=ids, past_key_values=ours)
    assert ours.get_seq_length() == int(want["len"]) == int(ids.shape[1] * (1 - ratio))
    for i, la in enumerate(ours.layers):
        close(_rows_signature(la.keys, la.values), want[f"sig{i}"], f"layer {i}")


def test_decoding_press_over_observed_attention_matches_the_reference(monkeypatch, ref):
    """DecodingPress(ObservedAttentionPress(), compression_interval=4, target_size=96): the compression scores with the
    current step's query only, as the reference's eager attentions of that step. One compression: the reference leaves
    the kept rows in score order and its divisor S - s follows the cache slots, so from a second compression on the two
    divisors see different rows (ours keep position order)."""
    cpu_backend.install(monkeypatch)
    observed_attention_backend.install(monkeypatch)
    ids = _ids(120)
    steps = [torch.tensor([[10 + t], [40 + t]]) for t in range(7)]

    def drive(model, cache, **fw):
        model.model(input_ids=ids, past_key_values=cache, **fw)
        lens = []
        for t, x in enumerate(steps):
            extra = {"cache_position": torch.tensor([ids.shape[1] + t])} if fw else {}
            model.model(input_ids=x, past_key_values=cache, **extra)
            lens.append(cache.get_seq_length())
        return lens

    def reference(kvpress):
        model, cache = _model("llama", "eager"), DynamicCache()
        with kvpress.DecodingPress(kvpress.ObservedAttentionPress(), compression_interval=4, target_size=96)(model):
            lens = drive(model, cache, cache_position=torch.arange(ids.shape[1]))
        return {"lens": np.array(lens), **_signatures(cache)}

    want = ref("decoding/observed", reference)
    model, cache = _model("llama", "eager"), DynamicCache()
    with DecodingPress(ObservedAttentionPress(), compression_interval=4, target_size=96)(model):
        lens = drive(model, cache)
    assert lens == [int(x) for x in want["lens"]] and cache.get_seq_length() == int(want["len"])
    for i, la in enumerate(cache.layers):
        close(_rows_signature(la.keys, la.values), want[f"sig{i}"], f"layer {i}")


def test_press_refuses_a_pruned_cache_and_a_narrow_sliding_window(monkeypatch):
    observed_attention_backend.install(monkeypatch)
    model = _model("qwen3", "sdpa")
    attn = model.model.layers[0].self_attn
    S, n_q = 12, 20
    keys = torch.randn(1, 2, S, 16)
    hidden = torch.randn(1, n_q, model.config.hidden_size)
    cos, sin = torch.ones(1, n_q, 16), torch.zeros(1, n_q, 16)
    press = ObservedAttentionPress(compression_ratio=0.5)
    with pytest.raises(ValueError, match="queries"):
        press.score(attn, hidden, keys, keys, None, {"position_embeddings": (cos, sin)})
    monkeypatch.setattr(attn, "sliding_window", 8, raising=False)
    with pytest.raises(NotImplementedError, match="sliding window"):
        press.score(attn, hidden[:, :S], keys, keys, None, {"position_embeddings": (cos[:, :S], sin[:, :S])})
    monkeypatch.setattr(attn, "sliding_window", S, raising=False)
    assert press.score(attn, hidden[:, :S], keys, keys, None,
                       {"position_embeddings": (cos[:, :S], sin[:, :S])}).shape == (1, 2, S)
