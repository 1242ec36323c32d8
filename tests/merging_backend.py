"""Float64 restatement of the MergingPress merge and oracle-backed stand-ins for `native.merging_compress` /
`native.merging_merge`, used by the merging tests next to tests/cpu_backend.py: the same contract (the definition of
include/kvpress_b200.h evaluated in float64, rounded once, ascending positions, lowest-position ties). Pure torch: they
run on CPU or CUDA tensors."""
import torch

from tests.cpu_backend import select_gather

EPS = 1e-6


def complement(kept: torch.Tensor, S: int) -> torch.Tensor:
    """The evicted positions [B, Hkv, S - n_kept] of ascending kept positions, ascending."""
    B, H, n_kept = kept.shape
    mask = torch.ones(B, H, S, dtype=torch.bool, device=kept.device)
    mask.scatter_(2, kept.long(), False)
    return mask.nonzero()[:, 2].reshape(B, H, S - n_kept)


def _rows(x: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    return x.gather(2, idx.long().unsqueeze(-1).expand(-1, -1, -1, x.shape[-1]))


def similarities64(keys: torch.Tensor, kept: torch.Tensor) -> torch.Tensor:
    """sim[b, j, e, t] in float64: the cosine similarity of evicted slot e and kept slot t, the norms clamped at 1e-6."""
    ev = complement(kept, keys.shape[2])
    kk, ke = _rows(keys.double(), kept), _rows(keys.double(), ev)
    nk, ne = kk.norm(dim=-1).clamp(min=EPS), ke.norm(dim=-1).clamp(min=EPS)
    return (ke @ kk.transpose(-1, -2)) / (ne.unsqueeze(-1) * nk.unsqueeze(-2))


def plan64(keys: torch.Tensor, kept: torch.Tensor):
    """(target, max_sim) [B, Hkv, n_evict]: torch.max over the kept slots, so ties and NaN go to the first column."""
    max_sim, target = similarities64(keys, kept).max(dim=-1)
    return target, max_sim


def gate(max_sim: torch.Tensor, similarity_threshold: float, merge_fraction: float) -> torch.Tensor:
    """ok [B, Hkv, n_evict]: the threshold, then the fraction gate by torch.quantile in max_sim's own dtype."""
    ok = max_sim >= similarity_threshold
    if merge_fraction < 1.0:
        thr = max_sim.masked_fill(~ok, float("-inf")).quantile(1.0 - merge_fraction, dim=-1, keepdim=True)
        ok = ok & (max_sim >= thr)
    return ok


def merged_values64(values: torch.Tensor, kept: torch.Tensor, target: torch.Tensor, max_sim: torch.Tensor,
                    ok: torch.Tensor) -> torch.Tensor:
    """The merged kept rows [B, Hkv, n_kept, D] in float64 from a merge plan; the unmerged rows are V[t] itself."""
    ev = complement(kept, values.shape[2])
    vk, ve = _rows(values.double(), kept), _rows(values.double(), ev)
    tn, en = vk.norm(dim=-1), ve.norm(dim=-1)
    w = max_sim.double().clamp(min=0) * ok.double()
    w = w * en / (en + tn.gather(2, target.long()) + EPS)
    acc_v = torch.zeros_like(vk).scatter_add_(2, target.long().unsqueeze(-1).expand_as(ve), w.unsqueeze(-1) * ve)
    acc_w = torch.zeros_like(tn).scatter_add_(2, target.long(), w)
    return torch.where((acc_w > 0).unsqueeze(-1), (vk + acc_v) / (1 + acc_w).unsqueeze(-1), vk)


def merge64(keys, values, kept, similarity_threshold, merge_fraction):
    """(merged kept rows in float64, target, max_sim) of ascending kept positions."""
    target, max_sim = plan64(keys, kept)
    ok = gate(max_sim, similarity_threshold, merge_fraction)
    return merged_values64(values, kept, target, max_sim, ok), target, max_sim


def merging_merge(keys, values, kept_idx, similarity_threshold, merge_fraction, return_plan=False):
    if kept_idx.shape[2] == 0:
        return values[:, :, :0].clone(), None, None
    v64, target, max_sim = merge64(keys, values, kept_idx, similarity_threshold, merge_fraction)
    plan = (target.to(torch.int32), max_sim.float()) if return_plan else (None, None)
    return (v64.to(values.dtype), *plan)


def merging_compress(scores, keys, values, similarity_threshold, merge_fraction, n_kept, return_indices=False,
                     return_plan=False):
    k_out, _, idx, _ = select_gather(scores.to(keys.dtype), keys, values, n_kept, True)
    v_out, target, sim = merging_merge(keys, values, idx, similarity_threshold, merge_fraction, return_plan)
    return k_out, v_out, (idx if return_indices else None), target, sim


def install(monkeypatch):
    from kvpress_b200 import native

    monkeypatch.setattr(native, "merging_compress", merging_compress)
    monkeypatch.setattr(native, "merging_merge", merging_merge)
