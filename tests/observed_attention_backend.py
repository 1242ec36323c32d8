"""CPU restatement of the ObservedAttention (H2O) score and oracle-backed stand-ins for
`native.observed_attention_score` / `native.observed_attention_compress`, used by the ObservedAttention tests next to
tests/cpu_backend.py: the same contract (float64 evaluation rounded once, the divisor S - s rounded to the cache
dtype, ascending positions, lowest-position ties). Pure torch: they run on CPU or CUDA tensors."""
import torch

from tests.cpu_backend import select_gather


def observed_attention_scores64(keys: torch.Tensor, q: torch.Tensor, scaling: float, block: int = 4096) -> torch.Tensor:
    """The library's definition (include/kvpress_b200.h, kvp_observed_attention_score) in float64, before the final
    rounding: with G = Hq / Hkv and query row i at position S - n_q + i,
    score[b,j,s] = (1/G) sum_g sum_i softmax_s(scaling q[b,jG+g,i] . k[b,j,s], causal)[s] / c(S - s), c(n) = n rounded
    to the cache dtype. Query rows are taken `block` at a time, so no n_q x S tensor exists beyond one block."""
    B, Hkv, S, D = keys.shape
    Hq, n_q = q.shape[1], q.shape[2]
    G, off = Hq // Hkv, S - n_q
    k = keys.double().unsqueeze(2)                                     # [B, Hkv, 1, S, D]
    qd = q.double().reshape(B, Hkv, G, n_q, D) * scaling
    pos = torch.arange(S, device=keys.device)
    col = torch.zeros((B, Hkv, S), dtype=torch.float64, device=keys.device)
    for i0 in range(0, n_q, block):
        i1 = min(n_q, i0 + block)
        y = torch.matmul(qd[:, :, :, i0:i1], k.transpose(-1, -2))     # [B, Hkv, G, rows, S]
        rows = torch.arange(off + i0, off + i1, device=keys.device)
        y.masked_fill_(pos[None, :] > rows[:, None], float("-inf"))
        col += torch.softmax(y, dim=-1).sum(dim=(2, 3))
    div = torch.arange(S, 0, -1, device=keys.device).to(keys.dtype).double()
    return col / (G * div)


def observed_attention_scores(keys: torch.Tensor, q: torch.Tensor, scaling: float) -> torch.Tensor:
    """observed_attention_scores64 rounded once to the cache dtype."""
    return observed_attention_scores64(keys, q.to(keys.dtype), scaling).to(keys.dtype)


def observed_attention_score(keys, q, scaling):
    return observed_attention_scores(keys, q, scaling)


def observed_attention_compress(keys, values, q, scaling, n_kept, return_indices=False, return_scores=False):
    scores = observed_attention_scores(keys, q, scaling)
    return select_gather(scores, keys, values, n_kept, return_indices, return_scores)


def install(monkeypatch):
    from kvpress_b200 import native, wide_head_scores

    monkeypatch.setattr(native, "observed_attention_score", observed_attention_score)
    monkeypatch.setattr(native, "observed_attention_compress", observed_attention_compress)
    # the stand-ins take any head_dim: the tiny CPU models (head_dim 16) stay on them
    monkeypatch.setattr(wide_head_scores, "observed_attention_on_tensor_cores", lambda *a: True)
