"""KVzapPress's surrogate scores and DMSPress's threshold eviction on the H100 (csrc/kvzap.cu), against the float64
definitions of tests/kvzap_backend.py."""
import pytest
import torch

from tests import kvzap_backend as KB

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]


def _model(hidden, hd, H, dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    w1 = (torch.randn(hd or H, hidden, generator=g) / hidden ** 0.5).to(dtype)
    b1 = (0.1 * torch.randn(hd or H, generator=g)).to(dtype)
    if hd == 0:
        return (w1, b1, None, None)
    w2 = (torch.randn(H, hd, generator=g) / hd ** 0.5).to(dtype)
    b2 = (0.1 * torch.randn(H, generator=g)).to(dtype)
    return (w1, b1, w2, b2)


def _cuda(ws):
    return tuple(None if w is None else w.cuda() for w in ws)


def _cache(B, H, S, dtype, D=64):
    k = torch.randn(B, H, S, D, device="cuda").to(dtype)
    return k, torch.randn_like(k)


def _tight(x, ws, scores):
    """Against an fp32 evaluation in another summation order: every score is within 1 ulp of it, or, where the sum
    cancels to far below its terms, within 2^-14 of the terms' magnitude (fp32 reordering moves a sum by a few 2^-24
    of it). Dropping a bias or replacing the GELU moves scores by percents of that magnitude."""
    ref32, mag = KB.fp32_scores(x, *_cuda(ws))
    d = KB.ulps_apart(scores, ref32.to(scores.dtype))
    ok = (d <= 1) | ((scores.float() - ref32).abs() <= 2.0 ** -14 * mag)
    assert ok.all(), (int((~ok).sum()), int(d.max()))


def _check(x, ws, scores):
    s64, E = KB.kvzap64(x.cpu(), *ws)
    ok = KB.within_bound(scores.cpu(), s64, E)
    assert ok.all(), (ok.numel() - ok.sum().item(), (scores.cpu().double() - s64).abs().max().item())
    _tight(x, ws, scores)


CASES = [  # (B, S, hidden, hd, Hkv)
    (1, 1, 4096, 512, 8), (1, 2, 4096, 512, 8), (2, 1, 1024, 64, 2), (1, 63, 4096, 512, 8), (1, 64, 1024, 1024, 16),
    (1, 65, 5120, 512, 8), (2, 1000, 4096, 512, 8), (1, 1000, 8192, 64, 1), (1, 1000, 1000, 512, 8),
    (1, 1000, 4096, 0, 8), (1, 63, 5120, 0, 16), (1, 1, 8192, 0, 1), (1, 1000, 4096, 1024, 2),
    (1, 32768, 4096, 512, 8), (1, 32768, 4096, 0, 8), (1, 300, 1024, 2048, 32), (1, 300, 16384, 8, 32),
]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,S,hidden,hd,H", CASES)
def test_score_within_the_documented_bound(dtype, B, S, hidden, hd, H):
    torch.manual_seed(S + hidden + hd)
    from kvpress_b200 import native

    x = torch.randn(B, S, hidden, device="cuda").to(dtype)
    ws = _model(hidden, hd, H, dtype)
    k, v = _cache(B, H, S, dtype)
    _check(x, ws, native.kvzap_score(x, k, v, _cuda(ws)))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("hd", [0, 512])
def test_score_at_128k(dtype, hd):
    from kvpress_b200 import native

    S, hidden, H = 131072, 4096, 8
    x = torch.randn(1, S, hidden, device="cuda").to(dtype)
    ws = _model(hidden, hd, H, dtype)
    k, v = _cache(1, H, S, dtype)
    scores = native.kvzap_score(x, k, v, _cuda(ws))
    sl = slice(0, S, 97)  # a float64 check of every 97th row keeps the host work small
    s64, E = KB.kvzap64(x[:, sl].cpu(), *ws)
    assert KB.within_bound(scores[..., sl].cpu(), s64, E).all()
    _tight(x, ws, scores)


@pytest.mark.parametrize("S", [1, 1000])
def test_repeatable_strided_and_rows_alone(S):
    from kvpress_b200 import native

    dtype, hidden, hd, H, B = torch.bfloat16, 1024, 256, 4, 2
    ws = _cuda(_model(hidden, hd, H, dtype))
    big = torch.randn(B, S, hidden + 64, device="cuda").to(dtype)
    x = big[..., 32:32 + hidden]  # a strided view
    k, v = _cache(B, H, S, dtype)
    a = native.kvzap_score(x, k, v, ws)
    b = native.kvzap_score(x.contiguous(), k, v, ws)
    assert torch.equal(a, b) and torch.equal(a, native.kvzap_score(x, k, v, ws))
    if S > 32:  # the same kernel for a row alone: the batch does not change it
        k1, v1 = k[1:], v[1:]
        assert torch.equal(native.kvzap_score(x[1:], k1, v1, ws), a[1:])


def test_graph_replay_and_poisoned_workspace():
    from kvpress_b200 import native

    dtype, hidden, hd, H, S = torch.float16, 2048, 512, 8, 777
    ws = _cuda(_model(hidden, hd, H, dtype))
    x = torch.randn(1, S, hidden, device="cuda").to(dtype)
    k, v = _cache(1, H, S, dtype)
    want = native.kvzap_score(x, k, v, ws)
    for buf in native._WS_CACHE.values():
        buf.fill_(0xFF)
    g = native.capture(lambda: native.kvzap_score(x, k, v, ws))
    assert torch.equal(g.replay(), want)
    out = native.kvzap_compress(x, k, v, ws, 400, return_indices=True, return_scores=True)
    assert torch.equal(out[3], want)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("hd", [0, 128])
def test_compress_selects_and_gathers(dtype, hd):
    from kvpress_b200 import native

    B, H, S, hidden, n_kept = 2, 4, 3000, 512, 1234
    ws = _cuda(_model(hidden, hd, H, dtype))
    x = torch.randn(B, S, hidden, device="cuda").to(dtype)
    k, v = _cache(B, H, S, dtype, D=128)
    k_out, v_out, idx, scores = native.kvzap_compress(x, k, v, ws, n_kept, return_indices=True, return_scores=True)
    assert torch.equal(scores, native.kvzap_score(x, k, v, ws))
    idx = idx.long()
    assert (idx.diff(dim=-1) > 0).all()
    kept = torch.gather(scores.float(), -1, idx)
    mask = torch.ones_like(scores, dtype=torch.bool).scatter_(-1, idx, False)
    dropped_max = scores.float().masked_fill(~mask, -float("inf")).amax(-1)
    assert (kept.amin(-1) >= dropped_max).all()
    gi = idx[..., None].expand(-1, -1, -1, 128)
    assert torch.equal(k_out, torch.gather(k, 2, gi)) and torch.equal(v_out, torch.gather(v, 2, gi))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("threshold", [0.0998, 0.0, -0.0, 1e-3, 1e5, float("inf"), -float("inf"), 0.1, 3.3333])
def test_eviction_is_torch_where(dtype, threshold):
    from kvpress_b200 import native

    torch.manual_seed(1)
    B, H, n = 2, 3, 5000
    base = torch.randn(B, H, n + 7, device="cuda").to(dtype)
    base[0, 0, :5] = torch.tensor([float("nan"), 0.0, -0.0, float("inf"), -float("inf")])
    base[1, 2, 10] = 0.099609375
    scores = base[..., 3:3 + n]  # strided rows
    for n_evict in (0, 1, 257, n - 1, n):
        got = native.threshold_evict(scores, n_evict, threshold, 17)
        want = KB.threshold_evict64(scores, n_evict, threshold, 17)
        assert all(torch.equal(g, w) for g, w in zip(got, want)), (threshold, n_evict)


def _tiny_llama():
    from tests.tiny_models import tiny_llama

    return tiny_llama(dtype=torch.bfloat16, device="cuda", head_dim=64)


def _kvzap(model, hd=64):
    from kvpress_b200 import KVzapConfig, KVzapModel, KVzapPress

    c = model.config
    torch.manual_seed(3)
    return KVzapPress(model_type="mlp", kvzap_model=KVzapModel(KVzapConfig(
        input_dim=c.hidden_size, output_dim=c.num_key_value_heads, hidden_dim=hd, n_modules=c.num_hidden_layers)))


@pytest.mark.parametrize("decoding", [False, True])
def test_dms_kvzap_masks_below_threshold(decoding):
    from transformers import DynamicCache

    from kvpress_b200 import DMSPress, KVPressTextGenerationPipeline
    from tests.tiny_models import word_tokenizer, words

    model = _tiny_llama()
    pipe = KVPressTextGenerationPipeline(model=model, tokenizer=word_tokenizer(), device="cuda")
    press = DMSPress(_kvzap(model), threshold=0.0, sliding_window_size=16, decoding=decoding)
    cache = DynamicCache()
    pipe(words(200, seed=1), question=words(6, seed=2), press=press, cache=cache, max_new_tokens=10)
    b, h, s = model.model.layers[0].self_attn.masked_key_indices
    assert 0 < press.compression_ratio < 1 and len(s) > 0
    assert len(set(zip(b.tolist(), h.tolist(), s.tolist()))) == len(s)
    with pytest.raises(ValueError) if decoding else _nothing():
        pipe(words(50, seed=1), questions=[words(3, seed=2), words(3, seed=3)], press=press, max_new_tokens=2)


class _nothing:
    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False


@pytest.mark.parametrize("wrap", ["kvzap", "adakv", "merging", "decoding"])
def test_wrappers_through_the_pipeline(wrap):
    from transformers import DynamicCache

    from kvpress_b200 import AdaKVPress, DecodingPress, KVPressTextGenerationPipeline, MergingPress
    from tests.tiny_models import word_tokenizer, words

    model = _tiny_llama()
    pipe = KVPressTextGenerationPipeline(model=model, tokenizer=word_tokenizer(), device="cuda")
    base = _kvzap(model)
    base.compression_ratio = 0.5
    if wrap == "decoding":
        # the buffered hidden states cover fewer positions than the cache: KVzap refuses to guess their scores
        press = DecodingPress(_kvzap(model), compression_interval=4, target_size=32)
        with pytest.raises(ValueError):
            pipe(words(120, seed=1), question=words(6, seed=2), press=press, max_new_tokens=10)
        return
    press = {"kvzap": base, "adakv": AdaKVPress(base), "merging": MergingPress(base)}[wrap]
    cache = DynamicCache()
    pipe(words(120, seed=1), question=words(6, seed=2), press=press, cache=cache, max_new_tokens=5)
    n = cache.layers[0].keys.shape[2]
    assert n < 125 if wrap != "adakv" else n >= 120


def test_unsupported_shapes_score_with_fp32_cublas(monkeypatch):
    """hidden not a multiple of 8, hd past 2048, more than 32 kv heads: KVzapPress scores with the torch fallback, within
    the documented bound, and compress selects on those scores."""
    from kvpress_b200 import KVzapConfig, KVzapModel, KVzapPress, native

    for hidden, hd, H in [(1004, 64, 2), (512, 2056, 2), (512, 0, 40)]:
        assert not native.kvzap_supported(hidden, hd, H)
        torch.manual_seed(hidden + hd)
        model = KVzapModel(KVzapConfig(input_dim=hidden, output_dim=H, hidden_dim=hd or None, n_modules=1))
        press = KVzapPress(kvzap_model=model, compression_ratio=0.5)
        x = torch.randn(1, 300, hidden, device="cuda").to(torch.bfloat16)
        k, v = _cache(1, H, 300, torch.bfloat16)
        layer = type("L", (torch.nn.Module,), {"layer_idx": 0})()
        scores = press.score(layer, x, k, v, None, {})
        ws = press.weights(0, k)
        s64, E = KB.kvzap64(x.cpu(), *(None if w is None else w.cpu() for w in ws))
        assert KB.within_bound(scores.cpu(), s64, E).all()
        k_out, _ = press.compress(layer, x, k, v, None, {})
        assert torch.equal(k_out, native.scores_compress(scores, k, v, 150)[0])


# --------------------------------------------------------------------------------------------------
# exact-size poisoned workspaces, and inputs and outputs past 4 GiB
# --------------------------------------------------------------------------------------------------
FAR = 4 << 30


def _far(nbytes, dtype, shape, offset=FAR):
    """A view of `shape` starting `offset` bytes into a fresh buffer, and the buffer."""
    buf = torch.empty(offset + nbytes + 256, dtype=torch.uint8, device="cuda")
    return buf[offset:offset + nbytes].view(dtype).view(*shape), buf


def _score_direct(x, k, ws, scores_out, n_kept=0, compress=None):
    """kvp_kvzap_score (or, with compress = (K_out, V_out, idx), kvp_kvzap_compress) on an exact-size workspace of
    0xFF bytes, writing into the caller's outputs."""
    from kvpress_b200 import native

    p = native.make_problem(k, k, n_kept)
    scorer = native.SCORER_KVZAP
    work = torch.full((native.workspace_bytes(p, scorer),), 0xFF, dtype=torch.uint8, device="cuda")
    args = native._kvzap_inputs(x, k, ws)
    name = "kvp_kvzap_score" if compress is None else "kvp_kvzap_compress"
    extra = (scores_out,) if compress is None else (k, k, *compress, scores_out)
    rc = getattr(native.load(), name)(native.ctypes.byref(p), *[native._ptr(a) if a is None or torch.is_tensor(a)
                                                                 else a for a in (*args, *extra)],
                                      work.data_ptr(), work.numel(), native._stream())
    assert rc == 0, rc


def _far_score(kind):
    from kvpress_b200 import native

    dtype, hidden, hd, H, S = torch.bfloat16, 1024, 256 if kind != "linear" else 0, 4, 700
    ws = _cuda(_model(hidden, hd, H, dtype))
    near = torch.randn(1, S, hidden, device="cuda").to(dtype)
    k, _ = _cache(1, H, S, dtype)
    want = native.kvzap_score(near, k, k, ws)
    x, xbuf = _far(near.numel() * 2, dtype, near.shape)
    x.copy_(near)
    out, obuf = _far(H * S * 2, dtype, (1, H, S))
    _score_direct(x, k, ws, out)
    assert torch.equal(out, want)
    del xbuf, obuf


def _far_compress():
    from kvpress_b200 import native

    dtype, hidden, hd, H, S, n_kept = torch.float16, 512, 128, 2, 900, 300
    ws = _cuda(_model(hidden, hd, H, dtype))
    x = torch.randn(1, S, hidden, device="cuda").to(dtype)
    near_k = torch.randn(1, H, S, 64, device="cuda").to(dtype)
    want = native.kvzap_compress(x, near_k, near_k, ws, n_kept, return_indices=True, return_scores=True)
    k, kbuf = _far(near_k.numel() * 2, dtype, near_k.shape)
    k.copy_(near_k)
    k_out, obuf = _far(H * n_kept * 64 * 2, dtype, (1, H, n_kept, 64))
    v_out = torch.empty_like(k_out)
    idx = torch.empty(1, H, n_kept, dtype=torch.int32, device="cuda")
    scores = torch.empty(1, H, S, dtype=dtype, device="cuda")
    _score_direct(x, k, ws, scores, n_kept, (k_out, v_out, idx))
    assert torch.equal(scores, want[3]) and torch.equal(idx, want[2]) and torch.equal(k_out, want[0])
    del kbuf, obuf


def _far_evict():
    from kvpress_b200 import native

    B, H, n, n_evict = 1, 4, 9000, 8900
    near = torch.randn(B, H, n, device="cuda").to(torch.bfloat16)
    want = KB.threshold_evict64(near, n_evict, 0.1, 3)
    sc, sbuf = _far(near.numel() * 2, torch.bfloat16, near.shape)
    sc.copy_(near)
    cap = B * H * n_evict
    out, obuf = _far(3 * cap * 8, torch.int64, (3, cap))
    count = torch.empty(1, dtype=torch.int64, device="cuda")
    work = torch.full((256 * 4,), 0xFF, dtype=torch.uint8, device="cuda")  # 8 B x 4 rows x 3 tiles -> 256 B needed
    sstride = (native.ctypes.c_int64 * 2)(H * n, n)
    rc = native.load().kvp_threshold_evict(0, B, H, n, sc.data_ptr(), sstride, n_evict, native.ctypes.c_float(0.1), 3,
                                           out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(), count.data_ptr(),
                                           work.data_ptr(), 256, native._stream())
    assert rc == 0, rc
    c = int(count.item())
    assert all(torch.equal(out[i, :c], want[i]) for i in range(3))
    del sbuf, obuf


FAR_CASES = {"kvp_kvzap_score": lambda: (_far_score("mlp"), _far_score("linear")),
             "kvp_kvzap_compress": _far_compress, "kvp_threshold_evict": _far_evict}


@pytest.mark.parametrize("name", sorted(FAR_CASES))
def test_inputs_and_outputs_past_4_gib_on_exact_poisoned_workspaces(name):
    FAR_CASES[name]()
    torch.cuda.empty_cache()


def test_every_kvzap_entry_point_has_a_far_offset_case():
    import re
    from pathlib import Path

    header = (Path(__file__).resolve().parent.parent / "include" / "kvpress_b200.h").read_text()
    names = set(re.findall(r"^kvp_status (kvp_kvzap_\w+|kvp_threshold_evict)\(", header, re.M))
    assert names == set(FAR_CASES)
