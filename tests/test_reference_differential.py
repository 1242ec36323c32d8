"""Differential test against the UNMODIFIED reference (NVIDIA/kvpress): the re-written presses, driven through the
same hooks on the same seeded random-init model, must retain the same rows as the reference presses.

What the reference computed in each case (row signatures of its compressed caches, cache lengths, masks, answers) is
stored in tests/golden/reference_differential.npz, so the comparison runs anywhere. To re-record it from a checkout of
the reference (located as in oracle/build_ref.py):  KVP_RECORD_REFERENCE=1 python -m pytest tests/test_reference_differential.py
The stored values come from another host's float32 CPU kernels: values compare with a tolerance of a few float32
rounding steps (a different retained row differs by orders of magnitude more); counts, lengths and masks exactly."""
import json
from pathlib import Path

import numpy as np
import pytest
import torch
from transformers import DynamicCache

from kvpress_b200 import ExpectedAttentionPress, KeyDiffPress, KnormPress, SnapKVPress, StreamingLLMPress
from tests import cpu_backend
from tests.support import TO_32BIT, close, ordered_signature, reference_store, rows_signature
from tests.tiny_models import distinct_ids, tiny_llama, tiny_qwen3

STORE = Path(__file__).resolve().parent / "golden" / "reference_differential.npz"
ref = reference_store(STORE, "KVP_RECORD_REFERENCE", TO_32BIT, merge=True)


def _signatures(cache) -> dict:
    return {f"sig{i}": rows_signature(la.keys, la.values) for i, la in enumerate(cache.layers)}


def _assert_signatures(cache, want: dict):
    for i, la in enumerate(cache.layers):
        close(rows_signature(la.keys, la.values), want[f"sig{i}"], f"layer {i}")


CASES = [
    ("knorm", lambda m: m.KnormPress, KnormPress, {}),
    ("streaming", lambda m: m.StreamingLLMPress, StreamingLLMPress, {"n_sink": 4}),
    ("snapkv", lambda m: m.SnapKVPress, SnapKVPress, {"window_size": 16, "kernel_size": 5}),
    ("expected_attention", lambda m: m.ExpectedAttentionPress, ExpectedAttentionPress, {"n_sink": 4}),
    ("keydiff", lambda m: m.KeyDiffPress, KeyDiffPress, {}),
    ("tova", lambda m: m.TOVAPress, __import__("kvpress_b200").TOVAPress, {}),
]


@pytest.mark.parametrize("name,ref_cls,our_cls,kw", CASES, ids=[c[0] for c in CASES])
@pytest.mark.parametrize("ratio", [0.25, 0.5, 0.7])
@pytest.mark.parametrize("family", ["llama", "qwen3"])
def test_same_rows_as_reference(monkeypatch, ref, name, ref_cls, our_cls, kw, ratio, family):
    cpu_backend.install(monkeypatch)
    model = tiny_llama() if family == "llama" else tiny_qwen3()
    ids = distinct_ids(160, seed=5)  # distinct tokens: no exactly tied layer-0 key norms
    S = ids.shape[1]

    def reference(kvpress):
        theirs = DynamicCache()
        with ref_cls(kvpress)(compression_ratio=ratio, **kw)(model):
            # transformers >= 5.5 no longer hands cache_position to attention; the reference hook needs it
            model.model(input_ids=ids, past_key_values=theirs, cache_position=torch.arange(S))
        out = {"len": theirs.get_seq_length()}
        for i, lt in enumerate(theirs.layers):
            out[f"norms{i}"] = lt.keys.norm(dim=-1).sort(-1).values
            out[f"sig{i}"] = rows_signature(lt.keys, lt.values)
        return out

    want = ref(f"same_rows/{name}/{ratio}/{family}", reference)
    ours = DynamicCache()
    with our_cls(compression_ratio=ratio, **kw)(model):
        model.model(input_ids=ids, past_key_values=ours)

    assert ours.get_seq_length() == int(want["len"]) == int(S * (1 - ratio))
    for i, lo in enumerate(ours.layers):
        if name == "knorm":
            # Qwen3's k_norm makes every key norm (nearly) equal: exact ties, broken differently by
            # torch.topk and by the lowest-position rule. The multiset of kept scores must still agree.
            close(lo.keys.norm(dim=-1).sort(-1).values, want[f"norms{i}"], f"layer {i}")
        else:
            close(rows_signature(lo.keys, lo.values), want[f"sig{i}"], f"layer {i}")


@pytest.mark.parametrize("inner", ["streaming", "snapkv"])
@pytest.mark.parametrize("family", ["llama", "qwen3"])
def test_key_rerotation_same_cache_as_reference(monkeypatch, ref, inner, family):
    """KeyRerotationPress (key_rerotation_press.py:133-152): the reference sorts the kept indices, so the
    compacted cache must agree ROW BY ROW, re-rotated keys included."""
    from kvpress_b200 import KeyRerotationPress

    cpu_backend.install(monkeypatch)
    model = tiny_llama() if family == "llama" else tiny_qwen3()
    ids = distinct_ids(160, seed=7)
    S, ratio = ids.shape[1], 0.4
    _, ref_cls, our_cls, kw = next(c for c in CASES if c[0] == inner)

    def reference(kvpress):
        theirs = DynamicCache()
        with kvpress.KeyRerotationPress(ref_cls(kvpress)(compression_ratio=ratio, **kw))(model):
            model.model(input_ids=ids, past_key_values=theirs, cache_position=torch.arange(S))
        out = {"len": theirs.get_seq_length()}
        for i, lt in enumerate(theirs.layers):
            out[f"keys{i}"], out[f"rows{i}"] = ordered_signature(lt.keys, lt.keys), ordered_signature(lt.keys, lt.values)
        return out

    want = ref(f"rerotation/{inner}/{family}", reference)
    ours = DynamicCache()
    press = KeyRerotationPress(our_cls(compression_ratio=ratio, **kw))
    assert press.compression_ratio == ratio
    with press(model):
        model.model(input_ids=ids, past_key_values=ours)

    assert ours.get_seq_length() == int(want["len"]) == int(S * (1 - ratio))
    for i, lo in enumerate(ours.layers):   # row by row, re-rotated keys included
        close(ordered_signature(lo.keys, lo.keys), want[f"keys{i}"], f"keys {i}")
        close(ordered_signature(lo.keys, lo.values), want[f"rows{i}"], f"rows {i}")


def _prefill(press, model, ids, reference=False):
    cache = DynamicCache()
    extra = {"cache_position": torch.arange(ids.shape[1])} if reference else {}
    with press(model):
        model.model(input_ids=ids, past_key_values=cache, **extra)
    return cache


def _reference_prefill(make_press, model, ids):
    """compute() for `ref`: the reference press's cache -> length, per-layer lengths and row signatures"""
    def compute(kvpress):
        cache = _prefill(make_press(kvpress), model, ids, reference=True)
        return {"len": cache.get_seq_length(), "lens": [la.keys.shape[2] for la in cache.layers], **_signatures(cache)}
    return compute


def _assert_same_rows(ours, want):
    assert [la.keys.shape[2] for la in ours.layers] == list(want["lens"])
    _assert_signatures(ours, want)


@pytest.mark.parametrize("ratio,beta", [(0.3, 20), (0.6, 4), (0.5, 1), (0.9, 20)])
def test_pyramidkv_same_rows_and_budgets_as_reference(monkeypatch, ref, ratio, beta):
    """pyramidkv_press.py:47-112: per-layer budgets (incl. the fallback branch) and the kept rows."""
    from kvpress_b200 import PyramidKVPress
    from kvpress_b200.presses.pyramidkv_press import pyramid_layer_budget

    cpu_backend.install(monkeypatch)
    model = tiny_llama(layers=4)
    ids = distinct_ids(160, seed=11)
    kw = dict(compression_ratio=ratio, window_size=16, kernel_size=5, beta=beta)
    from types import SimpleNamespace
    grid = [(q_len, r, b, layer) for q_len in (100, 777, 4096, 131072) for r in (0.1, 0.5, 0.75, 0.95)
            for b in (1, 5, 20) for layer in (0, 7, 31)]

    def reference(kvpress):
        out = _reference_prefill(lambda m: m.PyramidKVPress(**kw), model, ids)(kvpress)
        # the budget formula alone, over a grid, from the reference method
        out["budgets"] = [kvpress.PyramidKVPress(compression_ratio=r, window_size=64, beta=b).get_layer_budget(
            SimpleNamespace(config=SimpleNamespace(num_hidden_layers=32), layer_idx=layer), q_len)
            for q_len, r, b, layer in grid]
        return out

    want = ref(f"pyramidkv/{ratio}/{beta}", reference)
    ours = _prefill(PyramidKVPress(**kw), model, ids)
    lens = [layer.keys.shape[2] for layer in ours.layers]
    n_layers = model.config.num_hidden_layers
    assert lens == [pyramid_layer_budget(160, ratio, 16, beta, n_layers, i) for i in range(n_layers)]
    _assert_same_rows(ours, want)
    assert [pyramid_layer_budget(q_len, r, 64, b, 32, layer) for q_len, r, b, layer in grid] == list(want["budgets"])


@pytest.mark.parametrize("inner", ["knorm", "snapkv"])
@pytest.mark.parametrize("n_tokens,chunk", [(160, 40), (150, 64), (100, 256)])
def test_chunk_press_same_rows_as_reference(monkeypatch, ref, inner, n_tokens, chunk):
    from kvpress_b200 import ChunkPress

    cpu_backend.install(monkeypatch)
    model = tiny_llama()
    ids = distinct_ids(n_tokens, seed=12)
    _, ref_cls, our_cls, kw = next(c for c in CASES if c[0] == inner)
    if inner == "snapkv":
        kw = {"window_size": 8, "kernel_size": 3}
    want = ref(f"chunk/{inner}/{n_tokens}/{chunk}", _reference_prefill(
        lambda m: m.ChunkPress(ref_cls(m)(compression_ratio=0.5, **kw), chunk_length=chunk), model, ids))
    ours = _prefill(ChunkPress(our_cls(compression_ratio=0.5, **kw), chunk_length=chunk), model, ids)
    assert ours.get_seq_length() == int(want["len"])
    _assert_same_rows(ours, want)


def test_composed_and_per_layer_wrappers_same_rows_as_reference(monkeypatch, ref):
    from kvpress_b200 import ComposedPress, PerLayerCompressionPress

    cpu_backend.install(monkeypatch)
    model = tiny_llama()
    ids = distinct_ids(160, seed=13)
    # second press = Knorm: its scores do not depend on the ROW ORDER the first press leaves behind (the reference
    # emits top-k order, this package ascending positions; index-based scorers such as SnapKV's window or
    # StreamingLLM's sinks would read a different "last w rows" from the reference's permuted cache)
    ratios = [0.2, 0.6][: model.config.num_hidden_layers] + [0.5] * max(0, model.config.num_hidden_layers - 2)

    def composed(kvpress):
        rp = kvpress.ComposedPress([kvpress.SnapKVPress(0.25, window_size=16), kvpress.KnormPress(0.4)])
        return {**_reference_prefill(lambda m: rp, model, ids)(kvpress), "ratio": rp.compression_ratio}

    def per_layer(kvpress):
        rp = kvpress.PerLayerCompressionPress(kvpress.SnapKVPress(window_size=16), ratios)
        return {**_reference_prefill(lambda m: rp, model, ids)(kvpress), "ratio": rp.compression_ratio}

    want = ref("composed", composed)
    op = ComposedPress([SnapKVPress(0.25, window_size=16), KnormPress(0.4)])
    ours = _prefill(op, model, ids)
    assert ours.get_seq_length() == int(want["len"])
    assert op.compression_ratio == pytest.approx(float(want["ratio"]))
    _assert_same_rows(ours, want)

    want = ref("per_layer", per_layer)
    op = PerLayerCompressionPress(SnapKVPress(window_size=16), ratios)
    ours = _prefill(op, model, ids)
    assert op.compression_ratio == pytest.approx(float(want["ratio"]))
    with pytest.raises(AttributeError):
        op.compression_ratio = 0.1
    _assert_same_rows(ours, want)


def test_random_press_same_rows_as_reference_on_cpu(monkeypatch, ref):
    from kvpress_b200 import RandomPress

    cpu_backend.install(monkeypatch)
    model = tiny_llama()
    ids = distinct_ids(160, seed=14)
    want = ref("random", _reference_prefill(lambda m: m.RandomPress(0.5, seed=3), model, ids))
    _assert_same_rows(_prefill(RandomPress(0.5, seed=3), model, ids), want)


@pytest.mark.parametrize("inner", ["expected_attention", "snapkv"])
@pytest.mark.parametrize("alpha", [0.2, 0.0, 1.0])
def test_adakv_masks_the_same_keys_as_reference(monkeypatch, ref, inner, alpha):
    """adakv_press.py:53-78: per-head safeguard + bottom-k across heads; the pruned (batch, head, position)
    triples must be the reference's, and one decoding step through attention_patch must give the same output."""
    from kvpress_b200 import AdaKVPress

    cpu_backend.install(monkeypatch)
    model = tiny_llama()
    ids = distinct_ids(160, seed=21)
    S = ids.shape[1]
    _, ref_cls, our_cls, kw = next(c for c in CASES if c[0] == inner)
    attns = [layer.self_attn for layer in model.model.layers]

    def masks():
        out = []
        for a in attns:
            b, h, s = a.masked_key_indices
            out.append(sorted(zip(b.tolist(), h.tolist(), s.tolist())))
        return out

    def run(press, with_cache_position):
        cache = DynamicCache()
        with press(model):
            extra = {"cache_position": torch.arange(S)} if with_cache_position else {}
            model.model(input_ids=ids, past_key_values=cache, **extra)
            m = masks()
            extra = {"cache_position": torch.tensor([S])} if with_cache_position else {}
            step = model.model(input_ids=ids[:, :1], past_key_values=cache, **extra).last_hidden_state
        for a in attns:
            a.masked_key_indices = None
        return cache, m, step

    def reference(kvpress):
        c_ref, m_ref, y_ref = run(kvpress.AdaKVPress(ref_cls(kvpress)(compression_ratio=0.5, **kw), alpha_safeguard=alpha),
                                  True)
        return {"len": c_ref.get_seq_length(), "y": y_ref, **{f"mask{i}": np.array(m) for i, m in enumerate(m_ref)}}

    want = ref(f"adakv/{inner}/{alpha}", reference)
    c_our, m_our, y_our = run(AdaKVPress(our_cls(compression_ratio=0.5, **kw), alpha_safeguard=alpha), False)
    H = model.config.num_key_value_heads
    for i, a in enumerate(m_our):
        assert len(a) == ids.shape[0] * H * (S - int(S * 0.5))
        assert np.array_equal(np.array(a), want[f"mask{i}"])
    assert c_our.get_seq_length() == int(want["len"]) == S + 1      # AdaKV never shrinks the cache
    assert torch.allclose(y_our, torch.from_numpy(want["y"]), atol=1e-5)


@pytest.mark.parametrize("inner", ["knorm", "snapkv", "expected_attention"])
@pytest.mark.parametrize("n_tokens,chunk", [(160, 20), (150, 20), (150, 32), (15, 20)])
def test_chunkkv_press_same_rows_as_reference(monkeypatch, ref, inner, n_tokens, chunk):
    """chunkkv_press.py:52-117: whole chunks kept, ranked by head-summed mean score; ragged tail; S < chunk."""
    from kvpress_b200 import ChunkKVPress

    if inner != "knorm" and n_tokens < 32:
        pytest.skip("window scorers need more tokens than their window")
    cpu_backend.install(monkeypatch)
    model = tiny_llama()
    ids = distinct_ids(n_tokens, seed=31)
    _, ref_cls, our_cls, kw = next(c for c in CASES if c[0] == inner)
    if inner == "snapkv":
        kw = {"window_size": 8, "kernel_size": 3}
    def reference(kvpress):
        cache = _prefill(kvpress.ChunkKVPress(ref_cls(kvpress)(compression_ratio=0.4, **kw), chunk_length=chunk), model,
                         ids, reference=True)
        out = {"len": cache.get_seq_length(), "lens": [la.keys.shape[2] for la in cache.layers], **_signatures(cache)}
        for i, lt in enumerate(cache.layers):
            out[f"rows{i}"] = ordered_signature(lt.keys, lt.values)
        return out

    want = ref(f"chunkkv/{inner}/{n_tokens}/{chunk}", reference)
    ours = _prefill(ChunkKVPress(our_cls(compression_ratio=0.4, **kw), chunk_length=chunk), model, ids)
    assert ours.get_seq_length() == int(want["len"])
    if n_tokens < chunk:                               # plain press.compress: same rows, reference in top-k order
        _assert_same_rows(ours, want)
        return
    for i, lo in enumerate(ours.layers):               # both emit position order: caches are equal row by row
        close(ordered_signature(lo.keys, lo.values), want[f"rows{i}"], f"rows {i}")


@pytest.mark.parametrize("inner", ["knorm", "keydiff"])
@pytest.mark.parametrize("block_size", [16, 50, 400])
def test_block_press_same_rows_as_reference(monkeypatch, ref, inner, block_size):
    """block_press.py:49-98 incl. the reference's own invariant (tests/presses/test_block_press.py:30-63):
    a block at least as long as the context is the plain press."""
    from kvpress_b200 import BlockPress

    cpu_backend.install(monkeypatch)
    model = tiny_llama()
    ids = distinct_ids(160, seed=32)
    _, ref_cls, our_cls, kw = next(c for c in CASES if c[0] == inner)
    want = ref(f"block/{inner}/{block_size}", _reference_prefill(
        lambda m: m.BlockPress(ref_cls(m)(compression_ratio=0.5, **kw), block_size=block_size), model, ids))
    ours = _prefill(BlockPress(our_cls(compression_ratio=0.5, **kw), block_size=block_size), model, ids)
    _assert_same_rows(ours, want)
    if block_size >= ids.shape[1]:
        plain = _prefill(our_cls(compression_ratio=0.5, **kw), model, ids)
        _assert_same_rows(ours, {"lens": [la.keys.shape[2] for la in plain.layers], **_signatures(plain)})


def test_expected_attention_stats_press_same_rows_and_folder_layout_as_reference(monkeypatch, ref, tmp_path):
    """expected_attention_with_stats.py:21-110: stored (mu, Sigma) per layer instead of the per-prompt prologue;
    statistics folders are interchangeable with the reference's PyTorchModelHubMixin layout; the offline collector
    reproduces the reference formula (mean, unbiased covariance of the pre-RoPE queries beyond n_sink)."""
    from kvpress_b200 import ExpectedAttentionStatsPress
    from safetensors.torch import load_file

    from kvpress_b200.presses.expected_attention_with_stats import ExpectedAttentionStats, collect_query_statistics

    cpu_backend.install(monkeypatch)
    model = tiny_llama()
    cfg = model.config
    L, Hq, D = cfg.num_hidden_layers, cfg.num_attention_heads, cfg.head_dim
    batches = [distinct_ids(120, seed=40 + i, batch=1) for i in range(3)]
    stats = collect_query_statistics(model, batches, n_sink=4)
    # independent restatement of the reference's collect_queries arithmetic
    from kvpress_b200.utils import get_prerope_query_states
    qs = [[] for _ in range(L)]
    hooks = [layer.self_attn.register_forward_pre_hook(
        lambda m, a, kw, i=i: qs[i].append(get_prerope_query_states(m, kw["hidden_states"])[:, :, 4:]), with_kwargs=True)
        for i, layer in enumerate(model.model.layers)]
    with torch.no_grad():
        for ids in batches:
            model.model(input_ids=ids)
    for h in hooks:
        h.remove()
    for i in range(L):
        q = torch.cat(qs[i], dim=-2)[0]                                     # [Hq, N, D]
        mean = q.mean(dim=-2)
        c = q - mean.unsqueeze(-2)
        assert torch.allclose(stats.query_mean[i], mean, atol=1e-5)
        assert torch.allclose(stats.query_cov[i], c.transpose(-2, -1) @ c / (q.shape[-2] - 1), atol=1e-5)

    # folder layout: ours -> the reference's loader and writer (recorded: the folder the reference writes back);
    # that folder -> our loader; our folder has the reference's layout (same config, same tensor names and shapes)
    stats.save_pretrained(str(tmp_path / "ours"))
    ids = distinct_ids(160, seed=50)

    def reference(kvpress):
        from kvpress.presses.expected_attention_with_stats import ExpectedAttentionStats as RefStats

        theirs = RefStats.from_pretrained(str(tmp_path / "ours"))
        assert torch.equal(theirs.query_mean.data, stats.query_mean.data)
        assert torch.equal(theirs.query_cov.data, stats.query_cov.data)
        theirs.save_pretrained(str(tmp_path / "ref_folder"))
        files = sorted(f.name for f in (tmp_path / "ref_folder").iterdir())
        out = {"files": json.dumps(files), **{f"file:{f}": np.frombuffer((tmp_path / "ref_folder" / f).read_bytes(), np.uint8)
                                               for f in files}}
        # the presses, with and without covariance; hidden states are not needed
        for use_cov in (True, False):
            rp = kvpress.ExpectedAttentionStatsPress(compression_ratio=0.5, use_covariance=use_cov,
                                                     stats_folder=str(tmp_path / "ours"))
            cache = _prefill(rp, model, ids, reference=True)
            out.update({f"{use_cov}:{k}": v for k, v in _signatures(cache).items()})
            out[f"{use_cov}:lens"] = [la.keys.shape[2] for la in cache.layers]
            out[f"{use_cov}:mu"] = rp.mu
        return out

    want = ref("stats_press", reference)
    (tmp_path / "theirs").mkdir()
    for f in json.loads(str(want["files"])):
        (tmp_path / "theirs" / f).write_bytes(want[f"file:{f}"].tobytes())
    back = ExpectedAttentionStats.from_pretrained(str(tmp_path / "theirs"))
    close(back.query_cov.data, stats.query_cov.data, "query_cov")
    assert back.meta["n_sink"] == 4
    for f in json.loads(str(want["files"])):
        if f.endswith(".json"):
            assert json.loads((tmp_path / "ours" / f).read_text()) == json.loads((tmp_path / "theirs" / f).read_text())
        elif f.endswith(".safetensors"):
            mine, theirs = load_file(str(tmp_path / "ours" / f)), load_file(str(tmp_path / "theirs" / f))
            assert mine.keys() == theirs.keys()
            for k in mine:
                close(mine[k], theirs[k], k)

    for use_cov in (True, False):
        op = ExpectedAttentionStatsPress(compression_ratio=0.5, use_covariance=use_cov, stats_folder=str(tmp_path / "theirs"))
        o_cache = _prefill(op, model, ids)
        assert op.mu.shape == (L, Hq, D)
        close(op.mu, want[f"{use_cov}:mu"], "mu")
        _assert_same_rows(o_cache, {k.split(":", 1)[1]: v for k, v in want.items() if k.startswith(f"{use_cov}:")})
    assert ExpectedAttentionStatsPress.needs_hidden_states is False
    with pytest.raises(ValueError, match="No statistics given"):
        ExpectedAttentionStatsPress(0.5).post_init_from_model(model)


# ---------------------------------------------------------------------------------------------------------------------
# pipeline-level differentials (ADVICE r1): the reference pipeline driven on the same model, with a pre-hook that
# restores the `cache_position` kwarg transformers >= 5.3 no longer hands to attention modules (SURVEY F7)
# ---------------------------------------------------------------------------------------------------------------------
def _restore_cache_position(model):
    handles = []

    def pre(module, args, kwargs):
        if kwargs.get("cache_position") is None:
            past = kwargs["past_key_values"].get_seq_length(module.layer_idx)
            kwargs["cache_position"] = torch.arange(past, past + kwargs["hidden_states"].shape[1])
        return args, kwargs

    for layer in model.model.layers:
        handles.append(layer.self_attn.register_forward_pre_hook(pre, with_kwargs=True))
    return handles


def _pipeline(module, model):
    from tests.tiny_models import word_tokenizer

    return module.KVPressTextGenerationPipeline(model=model, tokenizer=word_tokenizer())


@pytest.mark.parametrize("family", ["llama", "qwen3"])
def test_pipeline_with_key_rerotation_matches_reference(monkeypatch, ref, family):
    """pipeline.py:231-232 of the reference: after KeyRerotationPress the question / answer positions continue from
    the COMPRESSED length. Same answers, and the positions the model sees are the reference's."""
    from kvpress_b200 import KeyRerotationPress
    from tests.tiny_models import words

    import kvpress_b200

    cpu_backend.install(monkeypatch)
    model = tiny_llama() if family == "llama" else tiny_qwen3()
    context, questions = words(150, seed=3), [words(4, seed=4), words(6, seed=5)]

    def run(module, handles):
        seen = []

        def pre(m, args, kwargs):
            if kwargs.get("position_ids") is not None:
                seen.append(kwargs["position_ids"].flatten().tolist())
        handles = handles + [model.model.register_forward_pre_hook(pre, with_kwargs=True)]
        try:
            out = _pipeline(module, model)(context, questions=questions, max_new_tokens=6, press=module.KeyRerotationPress(
                module.StreamingLLMPress(compression_ratio=0.4, n_sink=4)))
        finally:
            for h in handles:
                h.remove()
        return out["answers"], seen

    def reference(kvpress):
        answers, seen = run(kvpress, _restore_cache_position(model))
        return {"answers": np.array(answers), "seen": json.dumps(seen)}

    want = ref(f"pipeline_rerotation/{family}", reference)
    answers, seen = run(kvpress_b200, [])
    assert answers == [str(a) for a in want["answers"]]
    assert seen == json.loads(str(want["seen"])) and len(seen) > 2
    n_kept = int(151 * (1 - 0.4))
    assert seen[0][0] == n_kept          # the first question token sits right after the compacted cache


def test_decoding_press_with_stats_press_matches_reference(monkeypatch, ref, tmp_path):
    """DecodingPress(ExpectedAttentionStatsPress): the stats press reads only the LENGTH of the buffered hidden states
    (future RoPE positions); the zero-copy length-only buffer must reproduce the reference's concatenated buffer."""
    from kvpress_b200 import DecodingPress, ExpectedAttentionStatsPress
    from kvpress_b200.presses.expected_attention_with_stats import collect_query_statistics
    from tests.tiny_models import words

    cpu_backend.install(monkeypatch)
    model = tiny_llama()
    import kvpress_b200

    stats = collect_query_statistics(model, [distinct_ids(100, seed=60 + i, batch=1) for i in range(2)], n_sink=4)
    stats.save_pretrained(str(tmp_path / "stats"))
    context, question = words(60, seed=8), words(5, seed=9)
    kw = dict(compression_interval=7, target_size=40, hidden_states_buffer_size=256)
    # few future positions: the average RoPE rotation then depends visibly on where they start (q_len)
    skw = dict(stats_folder=str(tmp_path / "stats"), n_future_positions=3)

    def reference(kvpress):
        rp = kvpress.DecodingPress(base_press=kvpress.ExpectedAttentionStatsPress(**skw), **kw)
        cache = DynamicCache()
        handles = _restore_cache_position(model)
        try:
            theirs = _pipeline(kvpress, model)(context, question=question, max_new_tokens=24, press=rp, cache=cache)
        finally:
            for h in handles:
                h.remove()
        return {"answer": np.array(theirs["answer"]), "lens": [la.keys.shape[2] for la in cache.layers],
                **_signatures(cache)}

    want = ref("decoding_stats", reference)
    op = DecodingPress(base_press=ExpectedAttentionStatsPress(**skw), **kw)
    ours_cache = DynamicCache()
    ours = _pipeline(kvpress_b200, model)(context, question=question, max_new_tokens=24, press=op, cache=ours_cache)
    assert ours["answer"] == str(want["answer"])
    _assert_same_rows(ours_cache, want)
    assert not op.hidden_states_buffer and not op.hidden_states_lens     # reset on exit, nothing was cloned
