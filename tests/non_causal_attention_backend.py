"""Float64 restatement of the NonCausalAttention score and oracle-backed stand-ins for
`native.non_causal_attention_score` / `native.non_causal_attention_compress`, used by the NonCausalAttention tests next
to tests/cpu_backend.py: the same contract (float64 evaluation rounded once, ascending positions, lowest-position ties).
Pure torch: they run on CPU or CUDA tensors."""
import torch
import torch.nn.functional as F

from tests.cpu_backend import select_gather


def non_causal_attention_parts64(keys: torch.Tensor, values: torch.Tensor, q: torch.Tensor, chunk_size: int,
                                 block: int = 64, with_bound: bool = False):
    """x[b,j,s] = (1/G) sum_g A[b,jG+g,s] ||v[b,j,s]|| in float64 (include/kvpress_b200.h,
    kvp_non_causal_attention_score), with the last chunk padded as the reference pads it: padded keys at logit 0 (the
    reference's -1e-9), padded query rows all 0, hence uniform. `block` chunks at a time, so no S x S tensor exists.
    With `with_bound`, also tau[b,j,c]: the largest sum_d |q_d k_d| of any query head of kv head j over chunk c (the
    magnitude the kernel's fp32 error bound scales with, tests/test_gpu_non_causal_attention.py)."""
    B, Hkv, S, D = keys.shape
    G, cs = q.shape[1] // Hkv, int(chunk_size)
    n_chunks = -(-S // cs)
    pad = n_chunks * cs - S
    k = F.pad(keys.double(), (0, 0, 0, pad)).view(B, Hkv, 1, n_chunks, cs, D)
    qd = F.pad(q.to(keys.dtype).double(), (0, 0, 0, pad)).view(B, Hkv, G, n_chunks, cs, D)
    col = torch.empty((B, Hkv, n_chunks, cs), dtype=torch.float64, device=keys.device)
    tau = torch.empty((B, Hkv, n_chunks), dtype=torch.float64, device=keys.device) if with_bound else None
    for c0 in range(0, n_chunks, block):
        c1 = min(n_chunks, c0 + block)
        y = torch.matmul(qd[:, :, :, c0:c1], k[:, :, :, c0:c1].transpose(-1, -2))    # [B, Hkv, G, c, cs, cs]
        if pad and c1 == n_chunks:
            y[:, :, :, -1, cs - pad:] = 0
        col[:, :, c0:c1] = torch.softmax(y, dim=-1).sum(dim=-2).mean(dim=2)
        if with_bound:
            a = torch.matmul(qd[:, :, :, c0:c1].abs(), k[:, :, :, c0:c1].abs().transpose(-1, -2))
            tau[:, :, c0:c1] = a.amax(dim=(2, 4, 5))
    x = col.view(B, Hkv, n_chunks * cs)[..., :S] * values.double().norm(dim=-1)
    return (x, tau) if with_bound else x


def zscore64(x: torch.Tensor) -> torch.Tensor:
    """avg_pool1d(x, 3, padding 1) z-normalised over the whole tensor (unbiased std clamped at 1e-6), float64."""
    pooled = F.avg_pool1d(x, kernel_size=3, padding=1, stride=1)
    return (pooled - pooled.mean()) / pooled.std().clamp_min(1e-6)


def non_causal_attention_scores64(keys, values, q, chunk_size: int, block: int = 64) -> torch.Tensor:
    """The library's definition in float64, before the final rounding."""
    return zscore64(non_causal_attention_parts64(keys, values, q, chunk_size, block))


def non_causal_attention_score(keys, values, q, chunk_size):
    """non_causal_attention_scores64 rounded once to the cache dtype."""
    return non_causal_attention_scores64(keys, values, q, chunk_size).to(keys.dtype)


def non_causal_attention_compress(keys, values, q, chunk_size, n_kept, return_indices=False, return_scores=False):
    scores = non_causal_attention_score(keys, values, q, chunk_size)
    return select_gather(scores, keys, values, n_kept, return_indices, return_scores)


def install(monkeypatch):
    from kvpress_b200 import native, wide_head_scores

    monkeypatch.setattr(native, "non_causal_attention_score", non_causal_attention_score)
    monkeypatch.setattr(native, "non_causal_attention_compress", non_causal_attention_compress)
    # the stand-ins take any head_dim and chunk size: the tiny CPU models (head_dim 16) stay on them
    monkeypatch.setattr(wide_head_scores, "non_causal_attention_on_tensor_cores", lambda *a: True)
