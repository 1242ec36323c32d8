"""CPU restatement of the CriticalKV score and oracle-backed stand-ins for `native.criticalkv_score` /
`native.criticalkv_compress`, used by the CriticalKV tests next to tests/cpu_backend.py: the same contract (float64
evaluation rounded once, finfo.max on the n_first best base scores, ascending positions, lowest-position ties). Pure
torch: they run on CPU or CUDA tensors."""
import torch

from oracle import press_oracle as O
from tests.cpu_backend import select_gather


def criticalkv_scores(base: torch.Tensor, values: torch.Tensor, wo: torch.Tensor, epsilon: float,
                      n_first: int) -> torch.Tensor:
    """The library's definition (include/kvpress_b200.h, kvp_criticalkv_score), evaluated in float64 and rounded once
    to the cache dtype: with G = Hq / Hkv, norm[b,j,s] = mean over the G query heads h of kv head j of
    sum_n |v[b,j,s] . wo[n, h D:(h+1) D]|, score = (base + epsilon) * norm; then the n_first best base scores of every
    row (lowest-position ties) get finfo(dtype).max."""
    B, Hkv, S, D = values.shape
    Hq = wo.shape[1] // D
    G = Hq // Hkv
    w = wo.double().reshape(wo.shape[0], Hq, D)                                   # [hidden, Hq, D]
    v = O.repeat_kv(values.double(), G)                                           # [B, Hq, S, D]
    l1 = torch.einsum("bhsd,nhd->bhsn", v, w).abs().sum(-1)                       # [B, Hq, S]
    norm = l1.view(B, Hkv, G, S).mean(dim=2)
    scores = ((base.double() + epsilon) * norm).to(values.dtype)
    if n_first > 0:
        first = O.select_lowest_index_ties(base.to(values.dtype), n_first)
        scores.scatter_(-1, first, torch.finfo(scores.dtype).max)
    return scores


def criticalkv_score(base_scores, values, wo, epsilon, n_first):
    return criticalkv_scores(base_scores.to(values.dtype), values, wo.to(values.dtype), epsilon, n_first)


def criticalkv_compress(base_scores, keys, values, wo, epsilon, n_first, n_kept, return_indices=False,
                        return_scores=False):
    scores = criticalkv_score(base_scores, values, wo, epsilon, n_first)
    return select_gather(scores, keys, values, n_kept, return_indices, return_scores)


def install(monkeypatch):
    from kvpress_b200 import native, wide_head_scores

    monkeypatch.setattr(native, "criticalkv_score", criticalkv_score)
    monkeypatch.setattr(native, "criticalkv_compress", criticalkv_compress)
    # the stand-ins take any head_dim: the tiny CPU models (head_dim 16) stay on them
    monkeypatch.setattr(wide_head_scores, "criticalkv_on_tensor_cores", lambda *a: True)
