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
import math
from pathlib import Path

import numpy as np
import pytest
import torch
from transformers import DynamicCache

from kvpress_b200 import DecodingPress, ObservedAttentionPress, native
from tests import abi_cases, cpu_backend, observed_attention_backend
from tests.abi_cases import GOOD, ODD16
from tests.support import TO_32BIT, close, kv, rec, reference_store, rows_signature  # noqa: F401  (rec: fixture)
from tests.tiny_models import distinct_ids, tiny_model

STORE = Path(__file__).resolve().parent / "golden" / "observed_attention_reference.npz"

# --------------------------------------------------------------------------------------------------
# C ABI statuses
# --------------------------------------------------------------------------------------------------
def _align256(n: int) -> int:
    return (n + 255) // 256 * 256


def _checks(f, a, compress):
    """n_q -> scaling."""
    if not 1 <= a["n_q"] <= f["S"]:
        return -7
    return 0 if math.isfinite(a["scaling"]) and a["scaling"] > 0 else -7


def _short(f, a):
    """One byte short of the size for n_q = S: the per-row normalisers of fewer rows may still fit."""
    qrows = lambda n: _align256(4 * f["B"] * f["Hq"] * n)  # noqa: E731
    return -5 if qrows(a["n_q"]) == qrows(f["S"]) else -6


ABI = abi_cases.Spec(
    scorer=native.SCORER_OBSERVED_ATTENTION,
    slots={"kvp_observed_attention_score": "K q n_q scaling scores ws ws_bytes stream",
           "kvp_observed_attention_compress": "K V q n_q scaling K_out V_out idx scores ws ws_bytes stream"},
    valid=dict(K=GOOD, V=GOOD, q=GOOD, n_q=1000, scaling=0.125, K_out=GOOD, V_out=GOOD, idx=GOOD, scores=GOOD,
               ws=GOOD, ws_bytes="enough", stream=0),
    changes={
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
    },
    problem=("dtype", "S", "D", "Hq", "n_kept", "k_stride"),
    operands={"score": (["K", "q", "scores"], ["K", "q"]), "compress": (["q"], ["q"])},
    checks=_checks, short=_short)


def test_every_status_of_the_observed_attention_entry_points_follows_the_check_order():
    abi_cases.assert_statuses(__name__, 900)


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
    k, v = kv(B=2, H=2, S=64, D=64)
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
ref = reference_store(STORE, "KVP_RECORD_OBSERVED_ATTENTION", TO_32BIT)


def _signatures(cache) -> dict:
    return {"len": cache.get_seq_length(), **{f"sig{i}": rows_signature(la.keys, la.values)
                                               for i, la in enumerate(cache.layers)}}


@pytest.mark.parametrize("ratio", [0.25, 0.5, 0.7])
@pytest.mark.parametrize("family", ["llama", "qwen3"])
def test_observed_attention_keeps_the_reference_rows(monkeypatch, ref, ratio, family):
    cpu_backend.install(monkeypatch)
    observed_attention_backend.install(monkeypatch)
    ids = distinct_ids(160, seed=5)

    def reference(kvpress):
        model, cache = tiny_model(family, "eager"), DynamicCache()
        with kvpress.ObservedAttentionPress(compression_ratio=ratio)(model):
            model.model(input_ids=ids, past_key_values=cache, cache_position=torch.arange(ids.shape[1]))
        return _signatures(cache)

    want = ref(f"observed/{ratio}/{family}", reference)
    # same attention implementation as the reference, so that later layers see bit-equal hidden states; the press
    # ignores the eager weights it is handed
    model, ours = tiny_model(family, "eager"), DynamicCache()
    with ObservedAttentionPress(compression_ratio=ratio)(model):
        model.model(input_ids=ids, past_key_values=ours)
    assert ours.get_seq_length() == int(want["len"]) == int(ids.shape[1] * (1 - ratio))
    for i, la in enumerate(ours.layers):
        close(rows_signature(la.keys, la.values), want[f"sig{i}"], f"layer {i}")


def test_decoding_press_over_observed_attention_matches_the_reference(monkeypatch, ref):
    """DecodingPress(ObservedAttentionPress(), compression_interval=4, target_size=96): the compression scores with the
    current step's query only, as the reference's eager attentions of that step. One compression: the reference leaves
    the kept rows in score order and its divisor S - s follows the cache slots, so from a second compression on the two
    divisors see different rows (ours keep position order)."""
    cpu_backend.install(monkeypatch)
    observed_attention_backend.install(monkeypatch)
    ids = distinct_ids(120, seed=5)
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
        model, cache = tiny_model("llama", "eager"), DynamicCache()
        with kvpress.DecodingPress(kvpress.ObservedAttentionPress(), compression_interval=4, target_size=96)(model):
            lens = drive(model, cache, cache_position=torch.arange(ids.shape[1]))
        return {"lens": np.array(lens), **_signatures(cache)}

    want = ref("decoding/observed", reference)
    model, cache = tiny_model("llama", "eager"), DynamicCache()
    with DecodingPress(ObservedAttentionPress(), compression_interval=4, target_size=96)(model):
        lens = drive(model, cache)
    assert lens == [int(x) for x in want["lens"]] and cache.get_seq_length() == int(want["len"])
    for i, la in enumerate(cache.layers):
        close(rows_signature(la.keys, la.values), want[f"sig{i}"], f"layer {i}")


def test_press_refuses_a_pruned_cache_and_a_narrow_sliding_window(monkeypatch):
    observed_attention_backend.install(monkeypatch)
    model = tiny_model("qwen3", "sdpa")
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
