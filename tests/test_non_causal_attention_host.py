"""NonCausalAttention on the GPU-less box: the C ABI's checks of the two new entry points, the argument lists of their
wrappers, the float64 definition against the UNMODIFIED reference, and the press against the reference through the
oracle-backed stand-ins.

Statuses: every argument of kvp_non_causal_attention_score / kvp_non_causal_attention_compress made invalid on its own
(or set to another valid value), and every pair of such changes to two different arguments, against a restatement of the
documented check order (include/kvpress_b200.h). The pointers are fake, 16-byte aligned or not, and never dereferenced:
the calls run in a child process that sees no GPU, so a call that passes every check fails at its first CUDA call with
KVP_ERR_CUDA (-6).

Reference: what the reference's `NonCausalAttnPress.non_causal_chunked_attn` and `score` return on seeded float64 inputs,
and the rows its press keeps on the seeded tiny models, are stored in tests/golden/non_causal_attention_reference.npz.
To re-record them from a checkout of the reference (located as in oracle/build_ref.py):
    KVP_RECORD_NON_CAUSAL_ATTENTION=1 python -m pytest tests/test_non_causal_attention_host.py
"""
import ctypes
from pathlib import Path

import pytest
import torch
from transformers import DynamicCache

from kvpress_b200 import NonCausalAttnPress, native
from tests import abi_cases, cpu_backend, non_causal_attention_backend as NB
from tests.abi_cases import GOOD, ODD16
from tests.support import TO_INT32, kv, ordered_signature, rec, reference_store  # noqa: F401  (rec: fixture)
from tests.tiny_models import distinct_ids, tiny_llama, tiny_model

STORE = Path(__file__).resolve().parent / "golden" / "non_causal_attention_reference.npz"

# --------------------------------------------------------------------------------------------------
# C ABI statuses
# --------------------------------------------------------------------------------------------------
def _checks(f, a, compress):
    """chunk_size >= 1 -> shape instantiated."""
    if a["cs"] < 1:
        return -7
    return -2 if f["D"] not in (64, 128) or a["cs"] not in (128, 256) or not 1 <= f["Hq"] // f["Hkv"] <= 8 else 0


ABI = abi_cases.Spec(
    scorer=native.SCORER_NON_CAUSAL_ATTENTION,
    slots={"kvp_non_causal_attention_score": "K V q cs scores ws ws_bytes stream",
           "kvp_non_causal_attention_compress": "K V q cs K_out V_out idx scores ws ws_bytes stream"},
    valid=dict(K=GOOD, V=GOOD, q=GOOD, cs=256, K_out=GOOD, V_out=GOOD, idx=GOOD, scores=GOOD, ws=GOOD,
               ws_bytes="enough", stream=0),
    changes={
        "p": {"null": None},
        "dtype": {"3": 3},
        "S": {"0": 0},
        "D": {"12": 12, "64": 64, "96": 96},
        "Hq": {"5": 5, "32": 32},
        "n_kept": {"-1": -1, "0": 0, "1000": 1000},
        "v_stride": {"s100": (256000, 128000, 100)},
        "K": {"null": None, "odd": ODD16},
        "V": {"null": None, "odd": ODD16},
        "q": {"null": None, "odd": ODD16},
        "cs": {"0": 0, "-1": -1, "1": 1, "128": 128, "512": 512},
        "K_out": {"null": None},
        "V_out": {"null": None, "odd": ODD16},
        "idx": {"null": None},
        "scores": {"null": None},
        "ws": {"null": None, "odd": ODD16},
        "ws_bytes": {"short": "short"},
    },
    operands={"score": (["K", "V", "q", "scores"], ["K", "V", "q"]), "compress": (["q"], ["q"])},
    checks=_checks)


def test_every_status_of_the_non_causal_attention_entry_points_follows_the_check_order():
    abi_cases.assert_statuses(__name__, 800)


def test_workspace_and_launch_count_of_the_new_scorer_id():
    lib = native.load()
    p = native.KvpProblem()
    p.B, p.Hkv, p.Hq, p.D, p.n_kept, p.dtype = 1, 8, 32, 128, 0, 0
    prev = 0
    for S in (1, 2, 255, 256, 257, 4096, 16384, 131072):
        p.S = S
        nca, generic, n = ctypes.c_size_t(0), ctypes.c_size_t(0), ctypes.c_int(0)
        assert lib.kvp_workspace_bytes(ctypes.byref(p), native.SCORER_NON_CAUSAL_ATTENTION, ctypes.byref(nca)) == 0
        assert lib.kvp_workspace_bytes(ctypes.byref(p), native.SCORER_GENERIC, ctypes.byref(generic)) == 0
        # fp32 column sums and value norms of every position, fp64 partials per 256-position tile: nothing of cs x cs
        S_pad = -(-S // 256) * 256
        extra = nca.value - generic.value
        assert 2 * 8 * S_pad * 4 <= extra <= 2 * 8 * S_pad * 4 + 8 * S_pad // 256 * 16 + 4 * 256
        assert nca.value >= prev
        prev = nca.value
        assert lib.kvp_launches_per_compress(ctypes.byref(p), native.SCORER_NON_CAUSAL_ATTENTION, ctypes.byref(n)) == 0
        assert n.value == 6


# --------------------------------------------------------------------------------------------------
# wrappers: each argument after the kvp_problem, in order, down to the workspace and the stream
# --------------------------------------------------------------------------------------------------
def test_non_causal_attention_wrappers_pass_their_full_argument_list(rec, monkeypatch):  # noqa: F811
    workspaces = []
    real_workspace = native._workspace

    def spy(p, scorer, device):
        workspaces.append((scorer, real_workspace(p, scorer, device)))
        return workspaces[-1][1]

    monkeypatch.setattr(native, "_workspace", spy)
    P = lambda t: t.data_ptr()  # noqa: E731
    k, v = kv(B=2, H=2, S=64, D=64)
    q = torch.randn(2, 8, 64, 64).to(torch.bfloat16)

    def last(name, n_kept):
        got, p, a = rec.calls[-1]
        assert got == name and (p["n_kept"], p["Hq"], p["D"], p["S"]) == (n_kept, 8, 64, 64)
        s, ws = workspaces[-1]
        problem = native.make_problem(k, v, n_kept, 8)
        assert s == native.SCORER_NON_CAUSAL_ATTENTION
        assert a[-3:] == [ws.data_ptr(), native.workspace_bytes(problem, native.SCORER_NON_CAUSAL_ATTENTION), 0]
        return a[:-3]

    sc = native.non_causal_attention_score(k, v, q, 128)
    assert last("kvp_non_causal_attention_score", 0) == [P(k), P(v), P(q), 128, P(sc)]
    k_out, v_out, idx, sc = native.non_causal_attention_compress(k, v, q, 256, 20, return_indices=True,
                                                                 return_scores=True)
    assert last("kvp_non_causal_attention_compress", 20) == [P(k), P(v), P(q), 256, P(k_out), P(v_out), P(idx), P(sc)]
    qt = torch.randn(2, 64, 8, 64).to(torch.bfloat16).transpose(1, 2)  # a view: made contiguous
    native.non_causal_attention_compress(k, v, qt, 128, 20)
    a = last("kvp_non_causal_attention_compress", 20)
    assert a[2] != P(qt) and a[3] == 128 and a[6:] == [0, 0]
    # a [..., 8:-4, :] slice of the cache goes to the library in place, with its own strides
    ks, vs, qs = k[:, :, 8:-4], v[:, :, 8:-4], q[:, :, 8:-4]
    native.non_causal_attention_score(ks, vs, qs, 256)
    got, p, a = rec.calls[-1]
    assert a[:2] == [P(ks), P(vs)] and p["S"] == 52 and p["k_stride"] == (2 * 64 * 64, 64 * 64, 64)
    with pytest.raises(RuntimeError, match="prefill"):
        native.non_causal_attention_score(k, v, torch.randn(2, 8, 40, 64).to(torch.bfloat16), 256)
    with pytest.raises(RuntimeError, match="dtype"):
        native.non_causal_attention_score(k, v, q.half(), 256)


# --------------------------------------------------------------------------------------------------
# the float64 definition and the press against the unmodified reference
# --------------------------------------------------------------------------------------------------
ref = reference_store(STORE, "KVP_RECORD_NON_CAUSAL_ATTENTION", TO_INT32)


# (S, chunk_size, negative last chunk): one chunk, several, padded by 1 or more, not padded, a single position
DEFINITION = [(64, 32, False), (70, 32, False), (95, 32, False), (5, 256, False), (1, 256, False), (300, 256, False),
              (512, 256, False), (70, 32, True), (300, 256, True)]


def _definition_inputs(S, cs, negative):
    g = torch.Generator().manual_seed(S * 7 + cs)
    B, Hkv, G, D = 2, 2, 2, 16
    k = torch.randn(B, Hkv, S, D, generator=g, dtype=torch.float64) * 1.5
    v = torch.randn(B, Hkv, S, D, generator=g, dtype=torch.float64)
    q = torch.randn(B, Hkv * G, S, D, generator=g, dtype=torch.float64) * 1.5
    if negative:  # every logit of the last chunk's valid rows is -64: the padded keys take their mass
        s0 = (S - 1) // cs * cs
        k[:, :, s0:], q[:, :, s0:] = 2.0, -2.0
    return k, v, q


@pytest.mark.parametrize("S,cs,negative", DEFINITION, ids=[f"s{S}-cs{cs}{'-neg' if n else ''}" for S, cs, n in DEFINITION])
def test_float64_definition_is_the_reference(ref, S, cs, negative):
    """The column sums A and the z-scores of tests/non_causal_attention_backend.py against the reference's own
    non_causal_chunked_attn and score() on float64 inputs. The reference's softmax runs in fp32, so they agree to its
    rounding: 1e-6 of the largest value."""
    k, v, q = _definition_inputs(S, cs, negative)
    B, Hkv = k.shape[:2]
    G = q.shape[1] // Hkv

    def reference(kvpress):
        P = kvpress.presses.non_causal_attention_press.NonCausalAttnPress
        from transformers.models.llama.modeling_llama import repeat_kv
        A = P.non_causal_chunked_attn(q, repeat_kv(k, G), cs)
        model = tiny_llama(dtype=torch.float64, heads=4, kv_heads=2)
        attn = model.model.layers[0].self_attn
        hidden = torch.randn(B, S, model.config.hidden_size, generator=torch.Generator().manual_seed(S),
                             dtype=torch.float64)
        pos = model.model.rotary_emb(hidden, torch.arange(S)[None])
        kk, vv = k[:, :, :, :model.config.head_dim], v[:, :, :, :model.config.head_dim]
        z = P(compression_ratio=0.5, chunk_size=cs).score(attn, hidden, kk, vv, None, {"position_embeddings": pos})
        return {"A": A, "z": z}

    want = ref(f"definition/{S}/{cs}/{int(negative)}", reference)
    # A: the group mean of ours times ||v|| = 1 equals the mean over the group of the reference's per-head A
    ones = torch.full_like(v, 0.25)  # ||v|| = 1 at head_dim 16
    x = NB.non_causal_attention_parts64(k, ones, q, cs)
    A_ref = torch.as_tensor(want["A"], dtype=torch.float64).view(B, Hkv, G, S).mean(dim=2)
    assert torch.allclose(x, A_ref, rtol=1e-6, atol=1e-6 * float(A_ref.abs().max()))
    if negative:  # the padded query rows' pad / cs is nearly all the last chunk's keys receive
        s0 = (S - 1) // cs * cs
        pad = -(-S // cs) * cs - S
        assert torch.allclose(x[..., s0:], torch.full_like(x[..., s0:], pad / cs), rtol=1e-6)
    # z through our press's own query prologue on the same float64 module
    model = tiny_llama(dtype=torch.float64, heads=4, kv_heads=2)
    attn = model.model.layers[0].self_attn
    hidden = torch.randn(B, S, model.config.hidden_size, generator=torch.Generator().manual_seed(S), dtype=torch.float64)
    pos = model.model.rotary_emb(hidden, torch.arange(S)[None])
    kk, vv = k[:, :, :, :model.config.head_dim], v[:, :, :, :model.config.head_dim]
    qq = NonCausalAttnPress(chunk_size=cs).queries(attn, hidden, kk, {"position_embeddings": pos})
    z = NB.non_causal_attention_scores64(kk, vv, qq, cs)
    z_ref = torch.as_tensor(want["z"], dtype=torch.float64)
    if B * Hkv * S == 1:
        assert torch.isnan(z).all() and torch.isnan(z_ref).all()
    else:
        assert torch.allclose(z, z_ref, rtol=0, atol=1e-5 * float(z_ref.abs().max()))


def _kept_rows(cache) -> list:
    """Per layer, the ordered signature of every retained (K, V) row of every head."""
    return [ordered_signature(la.keys, la.values) for la in cache.layers]


def _shared_fraction(got: torch.Tensor, want: torch.Tensor) -> float:
    """Fraction of the retained rows of every head that both caches hold (signatures equal to float32 rounding)."""
    got, want = got.reshape(-1, got.shape[-1]), want.reshape(-1, want.shape[-1])
    hits = 0
    for a, b in zip(got, want):
        hits += int((torch.isclose(a[:, None], b[None, :], rtol=1e-5, atol=1e-6)).any(dim=1).sum())
    return hits / got.numel()


PRESS = [(ratio, family, cs, n) for ratio in (0.25, 0.5, 0.7) for family in ("llama", "qwen3")
         for cs, n in ((256, 160), (256, 240), (32, 160), (32, 150))]


@pytest.mark.parametrize("ratio,family,cs,n", PRESS, ids=[f"{f}-r{r}-cs{cs}-s{n}" for r, f, cs, n in PRESS])
def test_press_keeps_the_reference_rows(monkeypatch, ref, ratio, family, cs, n):
    """bf16 tiny models. The reference rounds the unscaled logits to bf16 before its softmax and the library does not,
    so scores near the selection threshold may order differently: at least 90 % of the kept rows are shared, and the
    cache lengths are equal."""
    cpu_backend.install(monkeypatch)
    NB.install(monkeypatch)
    ids = distinct_ids(n, seed=5)

    def model():
        return tiny_model(family, dtype=torch.bfloat16)

    def reference(kvpress):
        m, cache = model(), DynamicCache()
        with kvpress.NonCausalAttnPress(compression_ratio=ratio, chunk_size=cs)(m):
            m.model(input_ids=ids, past_key_values=cache, cache_position=torch.arange(ids.shape[1]))
        return {"len": cache.get_seq_length(),
                **{f"rows{i}": r.detach().float().numpy() for i, r in enumerate(_kept_rows(cache))}}

    want = ref(f"press/{ratio}/{family}/{cs}/{n}", reference)
    m, ours = model(), DynamicCache()
    with NonCausalAttnPress(compression_ratio=ratio, chunk_size=cs)(m):
        m.model(input_ids=ids, past_key_values=ours)
    assert ours.get_seq_length() == int(want["len"]) == int(n * (1 - ratio))
    for i, rows in enumerate(_kept_rows(ours)):
        frac = _shared_fraction(rows.float().double(), torch.as_tensor(want[f"rows{i}"], dtype=torch.float64))
        assert frac >= 0.9, f"layer {i}: {frac:.3f} of the kept rows shared"


def test_press_mirrors_the_reference_fields_and_asserts():
    press = NonCausalAttnPress()
    assert (press.compression_ratio, press.chunk_size) == (0.0, 256)
    m = tiny_llama()
    attn = m.model.layers[0].self_attn
    keys = torch.randn(1, 2, 12, 16)
    hidden = torch.randn(1, 10, m.config.hidden_size)
    pos = (torch.ones(1, 10, 16), torch.zeros(1, 10, 16))
    with pytest.raises(AssertionError, match="only supports prefill"):
        press.score(attn, hidden, keys, keys, None, {"position_embeddings": pos})
    with pytest.raises(AssertionError, match="chunk_size must be positive"):
        NonCausalAttnPress(chunk_size=0).score(attn, hidden[:, :10], keys[:, :, :10], keys[:, :, :10], None,
                                               {"position_embeddings": pos})
