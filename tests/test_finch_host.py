"""Finch on the GPU-less box: the C ABI's early checks of kvp_finch_score, kvp_finch_compress and
kvp_scores_compress_chunked (the statuses returned before the workspace is touched), the workspace formula and launch
count of scorer id 16, the unknown ids, the wrappers' argument lists, the host's chunk counts against the reference's
loop, and the press's argument and delimiter errors.
The pointers are fake and never dereferenced: every case here fails a check before any CUDA call.
"""
import ctypes
import re
from pathlib import Path

import numpy as np
import pytest
import torch
from transformers import DynamicCache

from kvpress_b200 import FinchPress, native

HEADER = Path(__file__).resolve().parent.parent / "include" / "kvpress_b200.h"
GOOD, ODD = 0x100000, 0x100008
OK, NULL, SHAPE, STRIDE, BAD = 0, -1, -2, -4, -7


def problem(B=1, H=2, Hq=8, S=1000, D=128, n_kept=500):
    p = native.KvpProblem()
    p.B, p.Hkv, p.Hq, p.S, p.D, p.n_kept, p.dtype = B, H, Hq, S, D, min(n_kept, S), 0
    for i, s in enumerate((H * S * D, S * D, D)):
        p.k_stride[i] = p.v_stride[i] = s
    return p


def align(x):
    return (x + 255) // 256 * 256


def finch_bytes(B, H, Hq, S, w):
    R, n_tiles = B * H, (S + 255) // 256
    S_pad = n_tiles * 256
    qpos = 128 if Hq == H else 64
    sel = [R * 1024, R * 1024, (3 * R + 64) * 4, R * n_tiles * 8, R * S_pad * 2, R * n_tiles * 264 * 2, R * 8]
    finch = [R * S * 4, B * Hq * (qpos * 64 + w) * 8, B * Hq * w * 4, R * S_pad * 4]
    return sum(align(x) for x in sel + finch)


def workspace_bytes(p, scorer=native.SCORER_FINCH):
    out = ctypes.c_size_t()
    assert native.load().kvp_workspace_bytes(ctypes.byref(p), scorer, ctypes.byref(out)) == 0
    return out.value


@pytest.mark.parametrize("B,H,Hq,S", [(1, 8, 32, 4096), (2, 2, 2, 1000), (1, 1, 8, 2), (3, 4, 12, 70000)])
def test_workspace_formula(B, H, Hq, S):
    assert workspace_bytes(problem(B, H, Hq, S)) == finch_bytes(B, H, Hq, S, max(1, S - 1))


def test_workspace_monotone_in_S():
    sizes = [workspace_bytes(problem(S=S)) for S in range(2, 3000, 37)]
    assert sizes == sorted(sizes)


def test_ids_and_launch_count():
    lib = native.load()
    n = ctypes.c_int()
    assert lib.kvp_launches_per_compress(ctypes.byref(problem()), 16, ctypes.byref(n)) == 0 and n.value == 6
    for unknown in (10, 12, 15):
        assert lib.kvp_launches_per_compress(ctypes.byref(problem()), unknown, ctypes.byref(n)) == BAD
    assert native.SCORER_FINCH == 16


def _params(name):
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    m = re.search(r"kvp_status\s+" + name + r"\(([^)]*)\)", text)
    return [a.strip() for a in m.group(1).split(",")]


@pytest.mark.parametrize("name", ["kvp_finch_score", "kvp_finch_compress", "kvp_scores_compress_chunked"])
def test_wrapper_argument_lists(name):
    restype, argtypes = native.SIGNATURES[name]
    params = _params(name)
    assert len(argtypes) == len(params)
    for t, decl in zip(argtypes, params):
        if "*" in decl or decl.startswith("kvp_stream_t"):
            assert t in (ctypes.c_void_p, native._PP, native._PI64), decl
        elif decl.startswith("size_t"):
            assert t is ctypes.c_size_t, decl
        else:
            assert t is ctypes.c_int32, decl


def score(p, K=GOOD, q=GOOD, w=40, normalize=1, out=GOOD):
    return native.load().kvp_finch_score(ctypes.byref(p) if p else None, K, q, w, normalize, out, None, 0, None)


def compress(p, K=GOOD, V=GOOD, q=GOOD, w=40, L=0, ck=0, tk=0, inv=None, Ko=GOOD, Vo=GOOD):
    return native.load().kvp_finch_compress(ctypes.byref(p) if p else None, K, V, q, w, 1, L, ck, tk, inv, Ko, Vo,
                                            None, None, None, 0, None)


def chunked(p, scores=GOOD, stride=True, L=256, ck=128, tk=116, inv=None, K=GOOD):
    st = (ctypes.c_int64 * 2)(0, 0) if stride else None
    return native.load().kvp_scores_compress_chunked(ctypes.byref(p) if p else None, scores, st, L, ck, tk, K, GOOD,
                                                     inv, GOOD, GOOD, None, None, 0, None)


def test_score_check_order():
    assert score(None) == NULL
    assert score(problem(D=12)) == SHAPE                          # validate first
    assert score(problem(), K=None, w=0) == NULL                  # null before alignment and window
    assert score(problem(), out=None) == NULL
    assert score(problem(), q=ODD, w=0) == STRIDE                 # alignment before window
    for w in (0, -1, 1000, 1001):
        assert score(problem(), w=w) == BAD
    assert score(problem(D=96), w=0) == BAD                       # window before the instantiation check
    assert score(problem(D=96)) == SHAPE
    assert score(problem(Hq=32)) == SHAPE                         # G = 16
    assert score(problem(), normalize=0) == NULL                  # every check passes: the workspace is null


def test_compress_check_order():
    assert compress(problem(n_kept=0), K=None, w=0) == OK          # n_kept == 0 short cut before the rest
    assert compress(problem(), V=None, q=None) == NULL
    assert compress(problem(), Ko=ODD, q=None) == STRIDE           # check_io before q_window
    assert compress(problem(), q=None, w=0) == NULL
    assert compress(problem(), q=ODD, w=0) == STRIDE
    assert compress(problem(), w=1000, L=-1) == BAD
    assert compress(problem(), L=-1) == BAD
    # S = 1000, L = 256: 3 full chunks and a tail of 232
    assert compress(problem(n_kept=3 * 128 + 116), L=256, ck=128, tk=116) == NULL  # workspace null: all passed
    assert compress(problem(n_kept=3 * 128 + 115), L=256, ck=128, tk=116) == BAD
    assert compress(problem(n_kept=3 * 257 + 116), L=256, ck=257, tk=116) == BAD  # chunk_kept > L
    assert compress(problem(n_kept=3 * 128 + 233), L=256, ck=128, tk=233) == BAD  # tail_kept > tail
    assert compress(problem(n_kept=3 * 128), L=256, ck=128, tk=0) == BAD          # a tail needs at least one
    assert compress(problem(n_kept=500), L=250, ck=125, tk=0) == NULL             # L divides S: no tail
    assert compress(problem(n_kept=600), L=2000, ck=0, tk=600) == NULL            # one short chunk
    assert compress(problem(D=96, n_kept=3 * 128 + 116), L=256, ck=128, tk=116, w=0) == BAD
    assert compress(problem(D=96, n_kept=3 * 128 + 116), L=256, ck=128, tk=116) == SHAPE


def test_scores_compress_chunked_check_order():
    assert chunked(problem(n_kept=0), scores=None, L=0) == OK
    assert chunked(problem(), K=None, scores=None) == NULL
    assert chunked(problem(), stride=False, L=0) == NULL
    assert chunked(problem(), L=0) == BAD
    assert chunked(problem(), tk=115) == BAD
    assert chunked(problem(D=120), inv=GOOD) == SHAPE
    assert chunked(problem(D=120)) == NULL                          # no inv_freq: every head_dim; workspace null
    assert chunked(problem(D=96), inv=GOOD) == NULL


@pytest.mark.parametrize("S,L,r", [(1000, 256, 0.5), (10, 5, 0.2), (17, 5, 0.2), (5, 7, 0.9), (4096, 4096, 0.5),
                                   (1031, 1, 0.3), (4097, 4096, 0.5)])
def test_chunk_counts_match_the_reference_loop(S, L, r):
    want = [max(1, int(min(L, S - i) * (1 - r))) for i in range(0, S, L)]  # finch_press.py's loop
    L_, ck, tk, n = native.chunk_counts(S, L, r)
    got = [ck] * (S // L) + ([tk] if S % L else [])
    assert L_ == L and got == want and n == sum(want)
    assert native.chunk_counts(S, None, r) == (0, 0, 0, int(S * (1 - r)))


class _Ids(torch.nn.Module):
    def forward(self, x):
        return x.float().unsqueeze(-1).expand(*x.shape, 3)


def test_press_errors_and_delimiter_hook():
    press = FinchPress(0.5)
    with pytest.raises(ValueError):
        with press(None):
            pass
    press.delimiter_token_id = 99
    emb = _Ids()
    ids = torch.tensor([[5, 6, 7, 99, 8, 9]])
    out = press.embed_token_forward_hook(emb, (ids,), emb(ids))
    assert press.window_size == 2 and out.shape[1] == 5 and 99 not in out[0, :, 0]
    with pytest.raises(AssertionError):
        press.embed_token_forward_hook(emb, (ids.repeat(2, 1),), emb(ids.repeat(2, 1)))
    two = torch.tensor([[5, 99, 7, 99, 8]])
    with pytest.raises(AssertionError):
        press.embed_token_forward_hook(emb, (two,), emb(two))
    last = torch.tensor([[5, 6, 99]])
    with pytest.raises(AssertionError):
        press.embed_token_forward_hook(emb, (last,), emb(last))
    keys = torch.zeros(1, 2, 8, 4)
    chunk = FinchPress(0.5, chunk_length=4)
    chunk.window_size = 2
    with pytest.raises(AssertionError):
        chunk.compress(None, None, keys, keys, None, {})
    wide = FinchPress(0.5)
    wide.window_size = 8
    with pytest.raises(ValueError):
        wide.compress(None, None, keys, keys, None, {})


# --------------------------------------------------------------------------------------------------
# the float64 definition and the press against the unmodified reference
# --------------------------------------------------------------------------------------------------
from tests import finch_backend as FB  # noqa: E402
from tests.support import TO_32BIT, close, ordered_signature, reference_store, rows_signature  # noqa: E402
from tests.tiny_models import tiny_model, word_tokenizer, words  # noqa: E402

STORE = Path(__file__).resolve().parent / "golden" / "finch_reference.npz"
ref = reference_store(STORE, "KVP_RECORD_FINCH", TO_32BIT)

# (name, S, w, ratio, chunk_length, normalize, rerotate). The window never has to share a chunk's budget: its positions
# all hold max + 1, and the reference's topk breaks such ties in no documented order (here: the lowest positions).
DEFINITION = [
    ("plain", 40, 6, 0.5, None, True, True),
    ("no-normalize", 40, 6, 0.5, None, False, True),
    ("no-rerotate", 33, 9, 0.3, None, True, False),
    ("chunked", 45, 5, 0.4, 12, True, True),  # the window fills the short last chunk's budget
    ("chunked-short-tail", 37, 2, 0.5, 8, False, False),
    ("window-1", 25, 1, 0.6, None, True, True),
]


def _definition_case(S, w):
    model = tiny_model()
    attn = model.model.layers[0].self_attn
    attn.rotary_emb = model.model.rotary_emb
    g = torch.Generator().manual_seed(S * 10 + w)
    hidden = torch.randn(2, S, model.config.hidden_size, generator=g)
    pe = model.model.rotary_emb(hidden, torch.arange(S).unsqueeze(0))
    keys = torch.randn(2, 2, S, 16, generator=g)
    values = torch.randn(2, 2, S, 16, generator=g)
    return attn, hidden, pe, keys, values


@pytest.mark.parametrize("name,S,w,ratio,L,normalize,rerotate", DEFINITION, ids=[d[0] for d in DEFINITION])
def test_float64_definition_is_the_reference(monkeypatch, ref, name, S, w, ratio, L, normalize, rerotate):
    """The float64 stand-in against the reference's own FinchPress.score and compress on float32 inputs: the scores (to
    float32 rounding, the window's max + 1 included) and the keys and values compress returns."""
    attn, hidden, pe, keys, values = _definition_case(S, w)

    def reference(kvpress):
        from kvpress.presses.finch_press import FinchPress as RefFinch

        press = RefFinch(compression_ratio=ratio, chunk_length=L, normalize_scores=normalize, rerotate_keys=rerotate)
        press.window_size = w
        scores = press.score(attn, hidden, keys, values, None, {"position_embeddings": pe})
        k, v = press.compress(attn, hidden, keys, values, None, {"position_embeddings": pe})
        return {"scores": scores, "keys": k, "values": v}

    want = ref(f"definition/{name}", reference)
    FB.install(monkeypatch)
    press = FinchPress(compression_ratio=ratio, chunk_length=L, normalize_scores=normalize, rerotate_keys=rerotate)
    press.window_size = w
    close(press.score(attn, hidden, keys, values, None, {"position_embeddings": pe}), want["scores"], name)
    k, v = press.compress(attn, hidden, keys, values, None, {"position_embeddings": pe})
    # the reference keeps its topk (score) order without re-rotation; with it, ascending positions as here
    sig = ordered_signature if rerotate else rows_signature
    close(sig(k, v), sig(torch.as_tensor(want["keys"]), torch.as_tensor(want["values"])), name)


# the reference's test_finch_press configurations, plus a longer prompt
PRESSES = {
    "r0.5": dict(compression_ratio=0.5),
    "no-rerotate": dict(compression_ratio=0.5, rerotate_keys=False),
    "no-normalize": dict(compression_ratio=0.5, normalize_scores=False),
    "chunk5": dict(compression_ratio=0.2, chunk_length=5),
}
# (tokens, position of the delimiter); chunk_length 5 needs w < 5 (1 - r) = 4
PROMPTS = {"short": (10, 8), "long": (90, 87)}


def _run_press(finch_cls, kw, family, prompt):
    model = tiny_model(family)
    n, at = PROMPTS[prompt]
    press = finch_cls(**kw)
    press.delimiter_token_id = model.config.eos_token_id
    ids = torch.arange(10, 10 + n)
    ids[at] = press.delimiter_token_id
    cache = DynamicCache()
    with press(model):
        # the delimiter's embedding is dropped: n - 1 positions reach the layers
        model.model(input_ids=ids.unsqueeze(0), past_key_values=cache, cache_position=torch.arange(n - 1))
    out = {"len": cache.get_seq_length(), "window": press.window_size}
    sig = ordered_signature if press.rerotate_keys else rows_signature
    for i, la in enumerate(cache.layers):
        out[f"sig{i}"] = sig(la.keys, la.values)
    return out


@pytest.mark.parametrize("prompt", sorted(PROMPTS))
@pytest.mark.parametrize("family", ["llama", "qwen3"])
@pytest.mark.parametrize("name", sorted(PRESSES))
def test_press_leaves_the_reference_cache(monkeypatch, ref, name, family, prompt):
    """The press on float32 tiny Llama / Qwen3 models, the delimiter detected and dropped by the embed_tokens hook: the
    same window size, cache length and kept (re-rotated) keys and values as the reference, to float32 rounding."""
    want = ref(f"press/{name}/{family}/{prompt}",
               lambda kvpress: _run_press(kvpress.FinchPress, PRESSES[name], family, prompt))
    FB.install(monkeypatch)
    got = _run_press(FinchPress, PRESSES[name], family, prompt)
    n, at = PROMPTS[prompt]
    assert got["window"] == int(want["window"]) == n - 1 - at
    assert got["len"] == int(want["len"])
    for i in range(2):
        close(got[f"sig{i}"], want[f"sig{i}"], f"{name} layer {i}")


def test_pipeline_with_the_delimiter(monkeypatch):
    """The text-generation pipeline with word_tokenizer() plus the added delimiter: the hook sets the window to the
    question's 12 tokens and drops the delimiter, and with rerotate_keys the answer's positions continue from the
    compressed length (the reference's pipeline.py:237), without it from the original one."""
    from kvpress_b200 import KVPressTextGenerationPipeline

    FB.install(monkeypatch)
    seen = []
    real = KVPressTextGenerationPipeline.generate_answer

    def spy(self, question_ids, cache, context_length, max_new_tokens):
        seen.append((context_length, cache.get_seq_length()))
        return real(self, question_ids, cache, context_length, max_new_tokens)

    monkeypatch.setattr(KVPressTextGenerationPipeline, "generate_answer", spy)
    for rerotate in (True, False):
        model, tok = tiny_model(), word_tokenizer()
        press = FinchPress(compression_ratio=0.5, rerotate_keys=rerotate)
        press.update_model_and_tokenizer(model, tok)
        assert press.delimiter_token_id == tok.convert_tokens_to_ids("<|finch_sep|>") == len(tok) - 1
        pipe = KVPressTextGenerationPipeline(model=model, tokenizer=tok, device="cpu")
        context = words(60, seed=1) + " <|finch_sep|> " + words(12, seed=3)
        n_ctx = len(tok(tok.bos_token + context)["input_ids"])  # the pipeline prepends BOS
        out = pipe(context, question=words(5, seed=2), press=press, max_new_tokens=4)
        assert isinstance(out["answer"], str) and press.window_size == 12
        context_length, cached = seen[-1]
        assert cached == int((n_ctx - 1) * 0.5)  # the delimiter dropped, then half of the positions kept
        assert context_length == (cached if rerotate else n_ctx)
