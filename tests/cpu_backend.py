"""Oracle-backed stand-in for `kvpress_b200.native`, used ONLY by the CPU host-logic tests.

The product has no CPU path (native.* raises on CPU tensors). To exercise the hook / pipeline /
DecodingPress plumbing on the GPU-less build box, tests monkeypatch the native entry points with these
functions, which implement the same contract (ascending positions, lowest-position ties) on top of
oracle/press_oracle.py.
"""
import torch

from oracle import press_oracle as O


def select_gather(scores, keys, values, n_kept, want_idx=True, want_scores=False):
    """The shared selection and compaction of a compress call: (K', V', idx or None, scores or None)."""
    idx = O.select_lowest_index_ties(scores, n_kept)
    k_out, v_out = O.gather_rows(keys, idx), O.gather_rows(values, idx)
    return k_out, v_out, (idx.to(torch.int32) if want_idx else None), (scores if want_scores else None)


def knorm_score(keys):
    return O.knorm_scores(keys)


def knorm_compress(keys, values, n_kept, return_indices=False, return_scores=False):
    return select_gather(O.knorm_scores(keys), keys, values, n_kept, return_indices, return_scores)


def streaming_score(keys, n_kept, n_sink):
    S = keys.shape[2]
    scores = torch.ones_like(keys[..., 0])
    scores[:, :, n_sink: n_sink + (S - n_kept)] = 0
    return scores


def streaming_compress(keys, values, n_kept, n_sink, return_indices=False):
    S = keys.shape[2]
    idx = O.streaming_kept(S, n_kept, n_sink).expand(keys.shape[0], keys.shape[1], -1)
    return O.gather_rows(keys, idx), O.gather_rows(values, idx), (idx.to(torch.int32) if return_indices else None)


def snapkv_score(keys, q_window, window, kernel_size):
    return O.snapkv_scores(q_window, keys, window, kernel_size)


def snapkv_compress(keys, values, q_window, window, kernel_size, n_kept, return_indices=False, return_scores=False):
    return select_gather(O.snapkv_scores(q_window, keys, window, kernel_size), keys, values, n_kept, return_indices,
                   return_scores)


def expected_attention_score(keys, values, mu, cov, epsilon, n_sink, use_vnorm):
    return O.expected_attention_scores(keys, values, mu, cov, epsilon, n_sink, use_vnorm)


def expected_attention_compress(keys, values, mu, cov, epsilon, n_sink, use_vnorm, n_kept, return_indices=False,
                                return_scores=False):
    scores = O.expected_attention_scores(keys, values, mu, cov, epsilon, n_sink, use_vnorm)
    return select_gather(scores, keys, values, n_kept, return_indices, return_scores)


def scores_compress(scores, keys, values, n_kept, return_indices=False):
    k_out, v_out, idx, _ = select_gather(scores, keys, values, n_kept, return_indices, False)
    return k_out, v_out, idx


def scores_compress_rerotate(scores, keys, values, n_kept, inv_freq, return_indices=False):
    idx = O.select_lowest_index_ties(scores, n_kept)
    k_out = O.rerotate_keys(keys, idx, inv_freq.float())
    return k_out, O.gather_rows(values, idx), (idx.to(torch.int32) if return_indices else None)


def keydiff_score(keys):
    return O.keydiff_scores(keys)


def keydiff_compress(keys, values, n_kept, return_indices=False, return_scores=False):
    return select_gather(O.keydiff_scores(keys), keys, values, n_kept, return_indices, return_scores)


def scores_select(scores, n_kept):
    return O.select_lowest_index_ties(scores, n_kept).to(torch.int32)


PATCHED = ["knorm_score", "knorm_compress", "streaming_score", "streaming_compress", "snapkv_score",
           "snapkv_compress", "expected_attention_score", "expected_attention_compress", "scores_compress", "scores_compress_rerotate", "scores_select", "keydiff_score", "keydiff_compress"]


def install(monkeypatch):
    from kvpress_b200 import native

    for name in PATCHED:
        monkeypatch.setattr(native, name, globals()[name])
    # the oracle-backed stand-ins take any head_dim / group size: the tiny CPU models (head_dim 16) stay on them
    from kvpress_b200 import wide_head_scores

    monkeypatch.setattr(wide_head_scores, "snapkv_on_tensor_cores", lambda *a: True)
    monkeypatch.setattr(wide_head_scores, "expected_attention_on_tensor_cores", lambda *a: True)
