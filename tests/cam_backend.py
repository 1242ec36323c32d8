"""Float64 restatement of the CaM compaction (kvp_cam_compress in include/kvpress_b200.h) and a stand-in for
`native.cam_compress`, next to tests/merging_backend.py. Pure torch: it runs on CPU or CUDA tensors.

The kept selection and the candidates depend only on the head mean m, which is computed exactly as the kernel computes
it (fp32 sum in ascending head order, / Hkv, one rounding), so both are exact. The draws are u < p_i with p_i in
float64, or, when the kernel's fp32 probabilities are given, u < those, so that a probability within fp32 rounding of u
cannot flip a decision."""
import torch

from oracle import press_oracle as O


def head_mean(scores: torch.Tensor) -> torch.Tensor:
    """m [B, S]: the fp32 sum of the Hkv scores in ascending head order, / Hkv, rounded once to the scores' dtype."""
    acc = scores[:, 0].float()
    for h in range(1, scores.shape[1]):
        acc = acc + scores[:, h].float()
    return (acc / scores.shape[1]).to(scores.dtype)


def plan(scores: torch.Tensor, n_kept: int, n_merge: int, merge_budget: int):
    """(kept [B, n_kept], candidates e [B, n_merge], t [B, n_merge], n [B, n_merge]), positions ascending."""
    B, _, S = scores.shape
    m = head_mean(scores)
    kept = O.select_lowest_index_ties(m.unsqueeze(1), n_kept)[:, 0].long()
    mask = torch.ones(B, S, dtype=torch.bool, device=m.device)
    mask.scatter_(1, kept, False)
    ev = mask.nonzero()[:, 1].reshape(B, S - n_kept)
    # (m descending, position descending), NaN first: the reference's flip + stable descending argsort
    order = m.gather(1, ev).flip(-1).argsort(dim=-1, descending=True, stable=True)[:, :n_merge]
    cand = ev.gather(1, ev.shape[1] - 1 - order).sort(dim=-1).values
    t = torch.searchsorted(kept, cand)
    n = (n_kept - t).clamp(max=merge_budget)
    return kept, cand, t, n


def cam64(scores, keys, values, attn_sum, n_merge, merge_budget, uniforms, n_kept, probs=None):
    """The definition in float64: (K_out, V_out float64, A_out, kept, candidates, p float64). `probs` (fp32
    [B, Hkv, n_merge]) replaces p_i in the draws when given."""
    B, H, S, D = keys.shape
    kept, cand, t, n = plan(scores, n_kept, n_merge, merge_budget)
    A = attn_sum.double()
    a_kept = A.gather(2, kept.unsqueeze(1).expand(B, H, n_kept))
    # window sums over the kept ranks [t_i, t_i + n_i), ascending, from a float64 running sum over the kept rows
    csum = torch.nn.functional.pad(a_kept.cumsum(-1), (1, 0))
    tt, nn_ = t.unsqueeze(1).expand(B, H, n_merge), n.unsqueeze(1).expand(B, H, n_merge)
    win = csum.gather(2, tt + nn_) - csum.gather(2, tt)
    p = A.gather(2, cand.unsqueeze(1).expand(B, H, n_merge)) / (win / nn_.clamp(min=1))
    p = torch.where(torch.isnan(p), torch.zeros_like(p), p)
    p = torch.where(torch.isposinf(p), torch.ones_like(p), p).clamp(0, 1)
    decide = p if probs is None else probs.double()
    w = (uniforms.double() < decide).double() / nn_.clamp(min=1)
    rows = lambda x, idx: x.gather(2, idx.view(B, 1, -1, 1).expand(B, H, idx.shape[1], D))  # noqa: E731
    k_out = rows(keys, kept)
    v_out = rows(values, kept).double()
    ve = rows(values, cand).double() * w.unsqueeze(-1)
    # candidate i adds to the kept ranks [t_i, t_i + n_i): a difference array, then a running sum over the ranks
    delta = torch.zeros(B, H, n_kept + 1, D, dtype=torch.float64, device=keys.device)
    delta.scatter_add_(2, tt.unsqueeze(-1).expand(B, H, n_merge, D), ve)
    delta.scatter_add_(2, (tt + nn_).unsqueeze(-1).expand(B, H, n_merge, D), -ve)
    v_out = v_out + delta[:, :, :n_kept].cumsum(2)
    return k_out, v_out, a_kept, kept, cand, p


def cam_compress(scores, keys, values, attn_sum, attn_out, n_merge, merge_budget, uniforms, n_kept,
                 return_indices=False, return_plan=False):
    B, H = keys.shape[:2]
    if uniforms is None:
        uniforms = torch.zeros(B, H, 0, device=keys.device)
    k_out, v64, a_out, kept, cand, p = cam64(scores.to(keys.dtype), keys, values, attn_sum, n_merge, merge_budget,
                                            uniforms, n_kept)
    attn_out.copy_(a_out)
    return (k_out, v64.to(values.dtype), kept.int() if return_indices else None,
            cand.int() if return_plan else None, p.float() if return_plan else None)


def install(monkeypatch):
    from kvpress_b200 import native

    monkeypatch.setattr(native, "cam_compress", cam_compress)
