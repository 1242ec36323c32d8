"""Host-side marshalling of kvpress_b200/native.py, checked on the GPU-less box: every wrapper is run on CPU tensors
against a recording stand-in for the shared library (the real library still answers kvp_workspace_bytes /
kvp_launches_per_compress, which need no device). What is pinned here: the kvp_problem fields and strides handed to
the C ABI for views, the pointers (views are consumed in place, small operands are made contiguous), dtype codes,
score strides for broadcast scores, NULL for optional operands, and the n_kept == 0 short cut."""
import pytest
import torch

from kvpress_b200 import native
from tests.support import kv, rec  # noqa: F401  (rec: fixture)


def test_strided_views_are_consumed_in_place(rec):
    wide_k = torch.randn(2, 6, 80, 64).to(torch.bfloat16)
    wide_v = torch.randn(2, 3, 100, 64).to(torch.bfloat16)
    k, v = wide_k[:, ::2, :50], wide_v[:, :, 10:60]              # every other head / a position window
    k_out, v_out, idx, scores = native.knorm_compress(k, v, 20, return_indices=True, return_scores=True)
    name, p, a = rec.calls[-1]
    assert name == "kvp_knorm_compress"
    assert (p["B"], p["Hkv"], p["Hq"], p["S"], p["D"], p["n_kept"], p["dtype"]) == (2, 3, 3, 50, 64, 20, 0)
    assert p["k_stride"] == (6 * 80 * 64, 2 * 80 * 64, 64) and p["v_stride"] == (3 * 100 * 64, 100 * 64, 64)
    assert a[0] == k.data_ptr() and a[1] == v.data_ptr()          # no copies
    assert a[2] == k_out.data_ptr() and a[3] == v_out.data_ptr() and a[4] == idx.data_ptr() and a[5] == scores.data_ptr()
    assert k_out.shape == (2, 3, 20, 64) and idx.dtype == torch.int32 and scores.shape == (2, 3, 50)
    assert a[7] >= 2 * 3 * 64 * 2                                  # workspace bytes from the real library


def test_layouts_the_kernels_cannot_address_are_copied_once(rec):
    k, v = kv()
    kt = k.transpose(2, 3).contiguous().transpose(2, 3)            # last dim strided: rows are not contiguous
    native.knorm_compress(kt, v, 10)
    _, p, a = rec.calls[-1]
    assert a[0] != kt.data_ptr() and p["k_stride"] == (3 * 50 * 64, 50 * 64, 64)
    odd = torch.randn(2, 3, 50, 64 + 4).to(torch.bfloat16)[..., 4:]   # rows not 16-byte aligned
    native.knorm_compress(odd, v, 10)
    assert rec.calls[-1][2][0] != odd.data_ptr()


def test_dtype_codes_single_row_and_empty_selection(rec):
    k, v = kv(dtype=torch.float16)
    native.knorm_compress(k, v, 5)
    assert rec.calls[-1][1]["dtype"] == 1
    k1, v1 = kv(S=1)
    native.streaming_compress(k1, v1, 1, 4)
    assert rec.calls[-1][1]["k_stride"][2] == 64                   # S == 1: the row stride stays addressable
    n = len(rec.calls)
    k_out, v_out, idx, _ = native.knorm_compress(k, v, 0, return_indices=True)
    assert len(rec.calls) == n and k_out.shape == (2, 3, 0, 64) and idx.shape == (2, 3, 0)   # nothing enqueued
    with pytest.raises(KeyError):
        native.make_problem(k.float(), v.float(), 1)               # dtypes other than bf16/fp16 have no code


def test_scorer_operands(rec):
    k, v = kv(B=2, H=2, S=200, D=128)
    q = torch.randn(2, 8, 16, 128).to(torch.bfloat16)
    native.snapkv_compress(k, v, q.transpose(1, 2).contiguous().transpose(1, 2), 16, 5, 100)
    name, p, a = rec.calls[-1]
    assert name == "kvp_snapkv_compress" and p["Hq"] == 8 and a[3:5] == [16, 5]
    mu_wide = torch.randn(2, 16, 128).to(torch.bfloat16)
    mu = mu_wide[:, ::2]                                            # non-contiguous small operand -> copied
    native.expected_attention_compress(k, v, mu, None, 0.25, 4, True, 60)
    name, p, a = rec.calls[-1]
    assert name == "kvp_expected_attention_compress" and p["Hq"] == 8
    assert a[2] != mu.data_ptr() and a[3] == 0                      # cov = NULL
    assert a[4] == pytest.approx(0.25) and a[5] == 4 and a[6] == 1
    with pytest.raises(RuntimeError, match="mu must be"):
        native.expected_attention_score(k, v, torch.zeros(2, 8, 64, dtype=torch.bfloat16), None, 0.0, 4, True)
    with pytest.raises(RuntimeError, match="q_window must be"):
        native.snapkv_score(k, q[:, :, :8], 16, 5)


def test_generic_scores_and_rerotation_operands(rec):
    k, v = kv(B=2, H=3, S=40, D=64)
    row = torch.rand(40).to(torch.bfloat16)                         # already in the cache dtype: stays a broadcast view
    native.scores_compress(row.expand(2, 3, 40), k, v, 10)          # broadcast scores: zero batch/head strides
    name, p, a = rec.calls[-1]
    assert name == "kvp_scores_compress" and a[1] == (0, 0)
    sc = torch.rand(2, 3, 40)
    native.scores_compress(sc, k, v, 10)
    assert rec.calls[-1][2][1] == (3 * 40, 40)
    inv_freq = torch.rand(32, dtype=torch.float64)
    native.scores_compress_rerotate(sc, k, v, 10, inv_freq)
    name, p, a = rec.calls[-1]
    assert name == "kvp_scores_compress_rerotate" and a[4] != inv_freq.data_ptr()    # converted to fp32
    with pytest.raises(RuntimeError, match="inv_freq"):
        native.scores_compress_rerotate(sc, k, v, 10, torch.rand(16))
    with pytest.raises(RuntimeError, match="scores must be"):
        native.scores_compress(sc[:, :2], k, v, 10)


# ---- the presses added late in round 1, driven through the REAL native wrappers (recording library) ---------------
class _Attn(torch.nn.Module):
    """Minimal attention module: what the presses read (head_dim, layer_idx, config, q_proj, rotary_emb)."""

    def __init__(self, hidden=64, heads=4, kv_heads=2, head_dim=16):
        super().__init__()
        from types import SimpleNamespace
        self.head_dim, self.layer_idx = head_dim, 0
        self.config = SimpleNamespace(num_attention_heads=heads, num_key_value_heads=kv_heads, num_hidden_layers=2,
                                      _attn_implementation="sdpa")
        self.q_proj = torch.nn.Linear(hidden, heads * head_dim, bias=False).to(torch.bfloat16)
        inv_freq = 1.0 / (10000.0 ** (torch.arange(0, head_dim, 2).float() / head_dim))

        def rotary(x, positions):
            ang = positions[..., None].float() * inv_freq
            emb = torch.cat((ang, ang), dim=-1)
            return emb.cos().to(x.dtype), emb.sin().to(x.dtype)
        self.rotary_emb = rotary
        self.rotary_emb.inv_freq = inv_freq


def _press_inputs(S=60):
    torch.manual_seed(0)
    attn = _Attn()
    hidden = torch.randn(2, S, 64).to(torch.bfloat16)
    keys, values = torch.randn(2, 2, S, 16).to(torch.bfloat16), torch.randn(2, 2, S, 16).to(torch.bfloat16)
    cos, sin = attn.rotary_emb(hidden, torch.arange(S)[None])
    return attn, hidden, keys, values, {"position_embeddings": (cos, sin)}


def test_tova_press_marshalling(rec):
    from kvpress_b200 import TOVAPress
    attn, hidden, keys, values, kwargs = _press_inputs()
    k2, v2 = TOVAPress(0.5).compress(attn, hidden, keys, values, None, kwargs)
    names = [c[0] for c in rec.calls]
    assert names == ["kvp_expected_attention_score", "kvp_scores_compress"]
    _, p, a = rec.calls[0]
    assert (p["B"], p["Hkv"], p["Hq"], p["S"], p["D"]) == (2, 2, 4, 60, 16)
    assert a[3] == 0 and a[5] == 0 and a[6] == 0            # no covariance, n_sink = 0, no value norms
    assert rec.calls[1][1]["n_kept"] == 30 and k2.shape == (2, 2, 30, 16)


def test_chunkkv_press_marshalling(rec):
    from kvpress_b200 import ChunkKVPress, KnormPress
    attn, hidden, keys, values, kwargs = _press_inputs(S=70)
    k2, _ = ChunkKVPress(KnormPress(0.5), chunk_length=20).compress(attn, hidden, keys, values, None, kwargs)
    names = [c[0] for c in rec.calls]
    assert names == ["kvp_knorm_score", "kvp_scores_compress"]
    _, p, a = rec.calls[1]
    assert a[1] == (0, 0)                                    # the 0/1 chunk mask is one broadcast row
    assert p["n_kept"] in (40, 30) and k2.shape[2] == p["n_kept"]   # 2 of 4 chunks: 2 full ones, or 1 full + the 10-token tail


def test_stats_press_marshalling(rec):
    from kvpress_b200 import ExpectedAttentionStatsPress
    attn, hidden, keys, values, kwargs = _press_inputs()
    press = ExpectedAttentionStatsPress(0.5)
    press.mu = torch.randn(2, 4, 16).to(torch.bfloat16)
    a_ = torch.randn(2, 4, 16, 16)
    press.cov = (a_ @ a_.transpose(-1, -2)).to(torch.bfloat16)
    press.compress(attn, hidden, keys, values, None, kwargs)
    name, p, a = rec.calls[-1]
    assert name == "kvp_expected_attention_compress" and p["Hq"] == 4 and a[3] != 0 and a[5] == 4
    press.use_covariance = False
    press.compress(attn, hidden, keys, values, None, kwargs)
    assert rec.calls[-1][2][3] == 0


class _CudaStandIn(torch.Tensor):
    """A CPU tensor that passes scores_select's CUDA check."""

    @property
    def is_cuda(self):
        return True


def test_every_wrapper_passes_its_full_argument_list(rec, monkeypatch):
    """All 13 wrappers: each argument after the kvp_problem, in order, down to the workspace and the stream."""
    workspaces = []
    real_workspace = native._workspace

    def spy(p, scorer, device):
        workspaces.append((scorer, real_workspace(p, scorer, device)))
        return workspaces[-1][1]

    monkeypatch.setattr(native, "_workspace", spy)

    def last(name, n_kept=0, Hq=2, scorer=None):
        """The last call's arguments; with `scorer`, its workspace (as the library sizes it) and the stream follow."""
        got, p, a = rec.calls[-1]
        assert got == name and (p["n_kept"], p["Hq"]) == (n_kept, Hq)
        if scorer is None:
            assert a[-1] == 0
            return a[:-1]
        s, ws = workspaces[-1]
        problem = native.make_problem(k, v, n_kept, Hq)
        assert s == scorer and a[-3:] == [ws.data_ptr(), native.workspace_bytes(problem, scorer), 0]
        return a[:-3]

    P = lambda t: t.data_ptr()  # noqa: E731
    k, v = kv(B=2, H=2, S=64, D=64)

    sc = native.knorm_score(k)
    assert last("kvp_knorm_score") == [P(k), P(sc)]
    k_out, v_out, idx, sc = native.knorm_compress(k, v, 20, return_indices=True, return_scores=True)
    assert last("kvp_knorm_compress", 20, scorer=native.SCORER_KNORM) == [P(k), P(v), P(k_out), P(v_out), P(idx), P(sc)]

    sc = native.keydiff_score(k)
    assert last("kvp_keydiff_score", scorer=native.SCORER_KEYDIFF) == [P(k), P(sc)]
    k_out, v_out, idx, _ = native.keydiff_compress(k, v, 20, return_indices=True)
    assert last("kvp_keydiff_compress", 20, scorer=native.SCORER_KEYDIFF) == [P(k), P(v), P(k_out), P(v_out), P(idx), 0]

    sc = native.streaming_score(k, 20, 4)
    assert last("kvp_streaming_score", 20) == [4, P(sc)]
    k_out, v_out, idx = native.streaming_compress(k, v, 20, 4, return_indices=True)
    assert last("kvp_streaming_compress", 20) == [4, P(k), P(v), P(k_out), P(v_out), P(idx)]

    q = torch.randn(2, 8, 16, 64).to(torch.bfloat16)
    sc = native.snapkv_score(k, q, 16, 5)
    assert last("kvp_snapkv_score", Hq=8, scorer=native.SCORER_SNAPKV) == [P(k), P(q), 16, 5, P(sc)]
    k_out, v_out, _, sc = native.snapkv_compress(k, v, q, 16, 5, 20, return_scores=True)
    assert last("kvp_snapkv_compress", 20, Hq=8, scorer=native.SCORER_SNAPKV) == \
        [P(k), P(v), P(q), 16, 5, P(k_out), P(v_out), 0, P(sc)]

    mu = torch.randn(2, 8, 64).to(torch.bfloat16)
    cov = torch.randn(2, 8, 64, 64).to(torch.bfloat16)
    sc = native.expected_attention_score(k, v, mu, cov, 0.5, 4, False)
    a = last("kvp_expected_attention_score", Hq=8, scorer=native.SCORER_EXPECTED_ATTENTION)
    assert a == [P(k), P(v), P(mu), P(cov), pytest.approx(0.5), 4, 0, P(sc)] and isinstance(a[4], float)
    k_out, v_out, idx, sc = native.expected_attention_compress(k, v, mu, None, 0.25, 4, True, 20, return_indices=True,
                                                               return_scores=True)
    assert last("kvp_expected_attention_compress", 20, Hq=8, scorer=native.SCORER_EXPECTED_ATTENTION) == \
        [P(k), P(v), P(mu), 0, 0.25, 4, 1, P(k_out), P(v_out), P(idx), P(sc)]

    scores = torch.rand(2, 2, 64).to(torch.bfloat16)
    k_out, v_out, idx = native.scores_compress(scores, k, v, 20, return_indices=True)
    assert last("kvp_scores_compress", 20, scorer=native.SCORER_GENERIC) == \
        [P(scores), (2 * 64, 64), P(k), P(v), P(k_out), P(v_out), P(idx)]
    inv_freq = torch.rand(32)
    k_out, v_out, _ = native.scores_compress_rerotate(scores, k, v, 20, inv_freq)
    assert last("kvp_scores_compress_rerotate", 20, scorer=native.SCORER_GENERIC) == \
        [P(scores), (2 * 64, 64), P(k), P(v), P(inv_freq), P(k_out), P(v_out), 0]

    wide = torch.rand(3, 4, 100).to(torch.float16)[:, 1:3, :50].as_subclass(_CudaStandIn)  # strided rows: in place
    idx = native.scores_select(wide, 10)
    name, p, a = rec.calls[-1]
    assert name == "kvp_scores_select" and idx.shape == (3, 2, 10) and idx.dtype == torch.int32
    assert (p["B"], p["Hkv"], p["Hq"], p["S"], p["D"], p["n_kept"], p["dtype"]) == (3, 2, 2, 50, 8, 10, 1)
    s, ws = workspaces[-1]
    assert s == native.SCORER_GENERIC
    assert a == [P(wide), (4 * 100, 100), P(idx), ws.data_ptr(), ws.numel(), 0]
