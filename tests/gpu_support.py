"""Helpers shared by the GPU tests: the library, the float64 references and input generators of the scorers, and the
bars their kernels are held to (each bar is described in the module docstring of the test file that states it)."""
import ctypes
import math
import re
from pathlib import Path

import torch
import torch.nn.functional as F
from transformers import DynamicCache

from oracle import press_oracle as O
from tests import non_causal_attention_backend as NB, observed_attention_backend as OB
from tests.conftest import ulp16_diff
from tests.tiny_models import distinct_ids, tiny_model

DEV = "cuda:0"


def _native():
    from kvpress_b200 import native
    native.load()
    return native


def _name(dtype) -> str:
    return "bf16" if dtype == torch.bfloat16 else "fp16"


def _sm_count() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def tiny_gpu_llama(head_dim=64):
    return tiny_model(dtype=torch.bfloat16, device=DEV, head_dim=head_dim, heads=8, kv_heads=2)


def gpu_ids(n=240):
    return distinct_ids(n, seed=11, device=DEV)


# ---------------------------------------------------------------------------------------------------
# the launchers' dispatch and schedule rules (expected_attention.cu: launch_ea_t, snapkv.cu: launch_snap_t)
# ---------------------------------------------------------------------------------------------------
def ea_instantiation(dtype, D: int, G: int):
    """<T, D, GR> of ea_logits_kernel: GR query heads resident per unit."""
    gr = 4 if G % 4 == 0 else (1 if G == 1 else 2)
    return (_name(dtype), D, gr)


def snap_parts(R: int, S: int, window: int, sm: int):
    """(ctas_per_row, parts holding tiles in pass 1, in pass 2) of launch_snap_t's row split."""
    n_tiles = (S + 127) // 128
    cpr = max(1, min(sm // R, n_tiles, 640))
    used = []
    for n in (n_tiles, min(n_tiles, (S - window + 127) // 128)):
        per = (n + cpr - 1) // cpr
        used.append((n + per - 1) // per)
    return cpr, used[0], used[1]


def ea_schedule(R: int, G: int, S: int):
    """CTA item ranges and per-unit (first CTA, CTA count) of the ExpectedAttention launch, from the library's own
    partition (kvp_debug_ea_pair_partition) and the launcher's worker count."""
    lib = ctypes.CDLL(str(_native().library_path()))
    fn = lib.kvp_debug_ea_pair_partition
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_int] * 5 + [ctypes.POINTER(ctypes.c_longlong)]
    gr = ea_instantiation(torch.bfloat16, 128, G)[2]
    n_units, n_tp = R * ((G + gr - 1) // gr), (S + 127) // 128
    n_workers = min(_sm_count(), 160, n_units * n_tp)
    out = (ctypes.c_longlong * 4)()
    ranges, spans = [], []
    for p in range(n_workers):
        assert fn(n_units, n_tp, n_workers, p, 0, out) == 0
        ranges.append((out[0], out[1]))
    for u in range(n_units):
        assert fn(n_units, n_tp, n_workers, 0, u, out) == 0
        spans.append((out[2], out[3]))
    return n_tp, n_workers, ranges, spans


UNIT_ROUNDOFF = {torch.bfloat16: 2.0 ** -7, torch.float16: 2.0 ** -10}


BIAS_MIN_N = 500


def ea_ref64(k, v, mu, cov, eps: float, n_sink: int, use_vnorm: bool) -> torch.Tensor:
    """expected_attention_scores_fp32 in float64, one (b, h) row at a time; forced positions are +inf."""
    B, H, S, D = k.shape
    G = mu.shape[1] // H
    eps = float(torch.tensor(eps, dtype=torch.float32))  # the kernel adds the fp32 epsilon
    out = torch.full((B, H, S), math.inf, dtype=torch.float64, device=k.device)
    for b in range(B):
        for h in range(H):
            kk = k[b, h, n_sink:].double()
            p = torch.zeros(S - n_sink, dtype=torch.float64, device=k.device)
            for g in range(G):
                hq = h * G + g
                logit = kk @ mu[b, hq].double() / math.sqrt(D)
                if cov is not None:
                    logit = logit + ((kk @ cov[b, hq].double()) * kk).sum(-1) / (2 * D)
                p += torch.softmax(logit, dim=-1)
            p /= G
            if use_vnorm:
                p = (p + eps) * v[b, h, n_sink:].double().norm(dim=-1)
            out[b, h, n_sink:] = p
    return out


def snap_ref64(q, k, window: int, kernel_size: int) -> torch.Tensor:
    """snapkv_scores_fp32 in float64, one (b, h) row at a time; the forced window is +inf. Window mean, box filter and
    group mean are linear, so the mean over all G * window rows is taken first."""
    B, H, S, D = k.shape
    G = q.shape[1] // H
    n = S - window
    out = torch.full((B, H, S), math.inf, dtype=torch.float64, device=k.device)
    i = torch.arange(G * window, device=k.device) % window
    mask = torch.arange(S, device=k.device)[None, :] > (S - window + i)[:, None]
    for b in range(B):
        for h in range(H):
            qq = q[b, h * G:(h + 1) * G].reshape(G * window, D).double()
            logits = (qq @ k[b, h].double().T) / math.sqrt(D)
            p = torch.softmax(logits.masked_fill(mask, -math.inf), dim=-1)[:, :n].mean(0)
            out[b, h, :n] = F.avg_pool1d(p[None, None], kernel_size, stride=1, padding=kernel_size // 2)[0, 0]
    return out


def assert_vs_ref64(got, ref, forced, what: str, ftz: bool = False, bias: bool = True) -> dict:
    """Bars 1-3 of the module docstring. got: [B, H, S] kernel scores; ref: float64 [B, H, S]; forced: bool [S]."""
    dtype = got.dtype
    ref = ref.to(got.device)
    forced = forced.to(got.device)
    g, r = got[..., ~forced], ref[..., ~forced]
    d = ulp16_diff(g, r.to(dtype))
    ok = d <= 1
    if ftz:  # ex2.approx.ftz: fp32 results below 2^-126 are flushed to zero
        ok |= (r < 2.0 ** -126) & (g == 0)
    assert ok.all(), f"{what}: {int((~ok).sum())} positions beyond 1 ulp of the fp64 score (max {int(d.max())})"
    stats = {"max_ulp": int(d.max()) if d.numel() else 0, "one_ulp": float((d == 1).float().mean()) if d.numel() else 0.0,
             "bias": 0.0}
    if bias:
        normal = r.abs() >= torch.finfo(dtype).tiny
        n = normal.sum(-1)
        rel = torch.where(normal, (g.double() - r) / r, torch.zeros_like(r))
        mean = rel.sum(-1) / n.clamp_min(1)
        bound = 8 * UNIT_ROUNDOFF[dtype] / torch.sqrt(12.0 * n.clamp_min(1).double())
        rows = n >= BIAS_MIN_N
        ratio = (mean.abs() / bound)[rows]
        if ratio.numel():
            stats["bias"] = float(ratio.max())
            assert (ratio <= 1).all(), f"{what}: row bias {float(ratio.max()):.1f}x its bound " \
                                       f"(mean rel error {float(mean[rows][ratio.argmax()]):.3e})"
    if forced.any():
        sentinel = (g.float().max() + 1).to(dtype)
        assert (got[..., forced] == sentinel).all(), f"{what}: forced positions are not round(max + 1)"
    print(f"[measured] {what}: max ulp {stats['max_ulp']}, 1-ulp fraction {stats['one_ulp']:.4f}, "
          f"worst row bias {stats['bias']:.3f} of the bound")
    return stats


def _gather(x, idx):
    return x.gather(2, idx.long().unsqueeze(-1).expand(-1, -1, -1, x.shape[-1]))


def assert_compress(k, v, k_out, v_out, idx, scores, n_kept: int):
    """Bar 4: the canonical selection of the kernel's own scores, and exact gathers."""
    want = O.select_lowest_index_ties(scores.cpu(), n_kept)
    assert torch.equal(idx.long().cpu(), want)
    assert torch.equal(k_out, _gather(k, idx)) and torch.equal(v_out, _gather(v, idx))


def _forced_head(S: int, n: int) -> torch.Tensor:
    m = torch.zeros(S, dtype=torch.bool)
    m[:n] = True
    return m


def _forced_tail(S: int, n: int) -> torch.Tensor:
    m = torch.zeros(S, dtype=torch.bool)
    m[S - n:] = True
    return m


def ea_inputs(B, H, G, S, D, dtype, seed, cov=True, mu_scale=0.5):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=gen, device=DEV)  # noqa: E731
    k, v = rn(B, H, S, D).to(dtype), rn(B, H, S, D).to(dtype)
    mu = (mu_scale * rn(B, H * G, D)).to(dtype)
    c = None
    if cov:
        a = rn(B, H * G, D, D) / D ** 0.5
        c = (a @ a.transpose(-1, -2)).to(dtype)
    return k, v, mu, c


def snap_inputs(B, H, G, S, D, window, dtype, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=gen, device=DEV)  # noqa: E731
    k, v = rn(B, H, S, D).to(dtype), rn(B, H, S, D).to(dtype)
    q = (1.5 * rn(B, H * G, window, D)).to(dtype)
    return k, v, q


def _layout(kind, B, H, S, D, dtype, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=gen, device=DEV).to(dtype)  # noqa: E731
    if kind == "slice_along_s":
        k, v = rn(B, H, S + 300, D)[:, :, 100:100 + S], rn(B, H, S + 50, D)[:, :, 50:]
    elif kind == "every_other_head":
        k, v = rn(B, 2 * H, S, D)[:, ::2], rn(B, 2 * H, S, D)[:, 1::2]
    elif kind == "transposed_bshd":
        k, v = rn(B, S, H, D).transpose(1, 2), rn(B, S, H, D).transpose(1, 2)
    elif kind == "one_head_of_wider_cache":
        k, v = rn(B, 4, S, D)[:, 2:3], rn(B, 3, S, D)[:, 1:2]
    else:  # "v_strided_k_contiguous"
        k, v = rn(B, H, S, D), rn(B, S, H, D).transpose(1, 2)
    return k, v


LAYOUTS = ["slice_along_s", "every_other_head", "transposed_bshd", "one_head_of_wider_cache", "v_strided_k_contiguous"]


def knorm_ref64(k: torch.Tensor) -> torch.Tensor:
    """-sqrt(sum k^2) in float64 on the device, one batch at a time."""
    return torch.stack([-(k[b].double() ** 2).sum(-1).sqrt() for b in range(k.shape[0])])


def _bits(x: torch.Tensor) -> torch.Tensor:
    return x.contiguous().view(torch.int16)


def _same(a, b) -> bool:
    """bitwise equal (None == None)"""
    if a is None or b is None:
        return a is None and b is None
    if a.dtype in (torch.bfloat16, torch.float16):
        return torch.equal(_bits(a), _bits(b))
    return torch.equal(a, b)


def ulp_at(z: torch.Tensor, dtype) -> torch.Tensor:
    """Spacing of the 16-bit dtype at |z| (its subnormal spacing below the normal range)."""
    mant, emin = (7, -126) if dtype == torch.bfloat16 else (10, -14)
    e = torch.floor(torch.log2(z.abs().clamp_min(2.0 ** emin)))
    return torch.exp2(e - mant)


def nca_inputs(B, Hkv, G, S, D, dtype, seed, negative_tail: bool = False):
    """Unscaled logits q.k of standard deviation about 6 (chunk maxima of 20-25, within the 10-100 of real layers) and
    value rows whose norms spread log-normally, as real caches' do (a near-constant ||v|| makes the z-score
    ill-conditioned: its std is then small against its mean). With `negative_tail`, every logit of the last chunk's
    valid rows is -D, so the padded keys take almost all of their mass."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    sig = 6 ** 0.5 / D ** 0.25
    k = (sig * torch.randn((B, Hkv, S, D), generator=g, device=DEV)).to(dtype)
    scale = torch.exp(0.7 * torch.randn((B, Hkv, S, 1), generator=g, device=DEV))
    v = (scale * torch.randn((B, Hkv, S, D), generator=g, device=DEV)).to(dtype)
    q = (sig * torch.randn((B, Hkv * G, S, D), generator=g, device=DEV)).to(dtype)
    if negative_tail:
        cs = 256
        s0 = (S - 1) // cs * cs
        k[:, :, s0:] = 1.0
        q[:, :, s0:] = -1.0
    return k, v, q


def nca_error_bound(x64, tau, z64, chunk_size: int, D: int, G: int) -> torch.Tensor:
    """E_s of the module docstring, per position."""
    B, Hkv, S = x64.shape
    cs = chunk_size
    gamma = (D + 1) * U32
    tau_s = tau.repeat_interleave(cs, dim=-1)[..., :S]
    dz = gamma * tau_s + 4 * U32 * tau_s + 2.0 ** -22 + cs * U32
    dp_rel = gamma * tau_s + dz + 4 * U32 * tau_s + 4 * U32 * math.log2(cs) + 2.0 ** -22
    eps_x = dp_rel + (cs * G + 2) * U32 + (D + 4) * U32
    pooled = F.avg_pool1d(x64, 3, padding=1, stride=1)
    dp = F.avg_pool1d(eps_x * x64.abs(), 3, padding=1, stride=1) + 3 * U32 * pooled.abs()
    e = float(eps_x.max()) + 3 * U32
    std = max(float(pooled.std()), 1e-6)
    d_mean = e * float(pooled.abs().mean())
    d_std = e * float(pooled.pow(2).mean().sqrt())
    return 1.01 * ((dp + d_mean) / std + z64.abs() * d_std / std)


def nca_ref(k, v, q, cs):
    B, Hkv, S, D = k.shape
    G = q.shape[1] // Hkv
    block = max(1, (1 << 25) // (B * q.shape[1] * cs * cs))
    x64, tau = NB.non_causal_attention_parts64(k, v, q, cs, block=block, with_bound=True)
    z64 = NB.zscore64(x64)
    return z64, nca_error_bound(x64, tau, z64, cs, D, G)


def oa_inputs(B, Hkv, G, S, n_q, D, dtype, seed, q_scale=1.5):
    g = torch.Generator(device=DEV).manual_seed(seed)
    k = torch.randn((B, Hkv, S, D), generator=g, device=DEV).to(dtype)
    v = torch.randn((B, Hkv, S, D), generator=g, device=DEV).to(dtype)
    q = (q_scale * torch.randn((B, Hkv * G, n_q, D), generator=g, device=DEV)).to(dtype)
    return k, v, q


def oa_ref64(k, q, scaling):
    B, Hkv, S, _ = k.shape
    block = max(1, (1 << 26) // (B * q.shape[1] * S))
    return OB.observed_attention_scores64(k, q, scaling, block=block)


def ckv_inputs(B, Hkv, G, S, D, hidden, dtype, seed, base_scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    v = torch.randn((B, Hkv, S, D), generator=g, device=DEV).to(dtype)
    wo = (torch.randn((hidden, Hkv * G * D), generator=g, device=DEV) / math.sqrt(D)).to(dtype)
    base = (torch.rand((B, Hkv, S), generator=g, device=DEV) * base_scale).to(dtype)
    return v, wo, base


def ckv_ref64(base, v, wo, eps: float) -> torch.Tensor:
    """(base + eps) * mean_g sum_n |v . wo[n, h D:(h+1) D]| in float64 on the device, one query head at a time."""
    B, Hkv, S, D = v.shape
    Hq = wo.shape[1] // D
    G = Hq // Hkv
    w = wo.double()
    norm = torch.zeros((B, Hkv, S), dtype=torch.float64, device=v.device)
    for h in range(Hq):
        for s0 in range(0, S, 4096):
            s1 = min(S, s0 + 4096)
            norm[:, h // G, s0:s1] += (v[:, h // G, s0:s1].double() @ w[:, h * D:(h + 1) * D].T).abs().sum(-1)
    return (base.double() + eps) * (norm / G)


def ckv_assert_scores(got, base, v, wo, eps, n_first, what, bias=True):
    dtype = got.dtype
    ref = ckv_ref64(base, v, wo, eps)
    forced = torch.zeros(got.shape, dtype=torch.bool, device=got.device)
    if n_first > 0:
        forced.scatter_(-1, O.select_lowest_index_ties(base, n_first), True)
    assert (got[forced] == torch.finfo(dtype).max).all(), f"{what}: forced positions do not hold finfo.max"
    if n_first > 0:  # no other position holds it (the fp64 scores of these inputs stay far below)
        assert int((got == torch.finfo(dtype).max).sum()) == int(forced.sum()), what
    g, r = got[~forced], ref[~forced]
    d = ulp16_diff(g, r.to(dtype))
    assert (d <= 1).all(), f"{what}: {int((d > 1).sum())} positions beyond 1 ulp of the fp64 score (max {int(d.max())})"
    worst = 0.0
    if bias:
        normal = (ref.abs() >= torch.finfo(dtype).tiny) & ~forced & torch.isfinite(ref.to(dtype))
        n = normal.sum(-1)
        rel = torch.where(normal, (got.double() - ref) / ref, torch.zeros_like(ref))
        mean = rel.sum(-1) / n.clamp_min(1)
        bound = 8 * UNIT_ROUNDOFF[dtype] / torch.sqrt(12.0 * n.clamp_min(1).double())
        rows = n >= BIAS_MIN_N
        ratio = (mean.abs() / bound)[rows]
        if ratio.numel():
            worst = float(ratio.max())
            assert (ratio <= 1).all(), f"{what}: row bias {worst:.2f}x its bound"
    print(f"[measured] {what}: max ulp {int(d.max()) if d.numel() else 0}, "
          f"1-ulp fraction {float((d == 1).float().mean()) if d.numel() else 0.0:.4f}, worst row bias {worst:.3f}")


def same16(a: torch.Tensor, b: torch.Tensor) -> bool:
    """Bitwise equality of two 16-bit tensors (torch.equal is False wherever both hold NaN)."""
    return a.shape == b.shape and torch.equal(a.view(torch.int16), b.view(torch.int16))


def lagkv_inputs(B, H, S, D, dtype, seed, scale=1.0):
    """Gaussian K and V, with a per-row scale that spreads log-normally (the rows of a real cache differ in norm)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    k = (scale * torch.exp(0.3 * torch.randn((B, H, S, 1), generator=g, device=DEV))
         * torch.randn((B, H, S, D), generator=g, device=DEV)).to(dtype)
    v = (scale * torch.exp(0.3 * torch.randn((B, H, S, 1), generator=g, device=DEV))
         * torch.randn((B, H, S, D), generator=g, device=DEV)).to(dtype)
    return k, v


def _prefill(ids):
    return lambda model, cache: model.model(input_ids=ids, past_key_values=cache)


def _shared(a: DynamicCache, b: DynamicCache) -> float:
    """Fraction of the value rows of `a` that `b` holds too, per head (values are gathered as they are under every
    press, keys may be re-rotated)."""
    hits = total = 0
    for la, lb in zip(a.layers, b.layers):
        va, vb = la.values.float(), lb.values.float()
        same = (va[..., :, None, :] == vb[..., None, :, :]).all(dim=-1).any(dim=-1)
        hits, total = hits + int(same.sum()), total + same.numel()
    return hits / total


def _masked(model) -> list:
    """Per layer, the set of (b, h, s) an AdaKVPress masked."""
    return [set(zip(*(t.tolist() for t in layer.self_attn.masked_key_indices))) for layer in model.model.layers]


MANT_BITS = {torch.bfloat16: 7, torch.float16: 10}
MIN_EXP = {torch.bfloat16: -126, torch.float16: -14}
U32 = 2.0 ** -24


E_SCALE_FRACTION = 2.0 ** -8  # max E_s of a row, as a share of its largest |score|


def ulp16(x: torch.Tensor) -> torch.Tensor:
    """float64 spacing of x's 16-bit format at |x|"""
    e = torch.floor(torch.log2(x.double().abs())).clamp_min(MIN_EXP[x.dtype])
    return torch.exp2(e - MANT_BITS[x.dtype])


def _ulp32(x: torch.Tensor) -> torch.Tensor:
    return torch.exp2(torch.floor(torch.log2(x.abs())).clamp_min(-126) - 23)


MERGE_THREADS = 1024  # kKdMergeThreads


CHUNK = 256  # kScoreChunk: positions per anchor / score CTA


# kLanesPerRow of csrc/common.cuh: the lanes-per-row counts the CUDA-core score kernels are instantiated for
LANES_PER_ROW = tuple(int(x) for x in re.search(
    r"constexpr int kLanesPerRow\[\] = \{([\d, ]+)\};",
    (Path(__file__).resolve().parent.parent / "kvpress_b200" / "csrc" / "common.cuh").read_text()).group(1).split(","))


def lanes_per_row(D: int) -> int:
    """The LPR with_lanes_per_row picks for head_dim D: the first kLanesPerRow entry >= D / 8, else the last."""
    return next((lpr for lpr in LANES_PER_ROW if D // 8 <= lpr), LANES_PER_ROW[-1])


def kd_dpad(D: int) -> int:
    return 32 if D <= 32 else 64 if D <= 64 else 128 if D <= 128 else 256


def kd_groups(D: int) -> int:
    """G of keydiff_merge_kernel"""
    return MERGE_THREADS // kd_dpad(D)


def kd_chunks(S: int) -> int:
    return (S + CHUNK - 1) // CHUNK


def kd_chain(S: int, D: int) -> int:
    """L: the longest addition chain of an anchor component (see the module docstring)"""
    lpr, G = lanes_per_row(D), kd_groups(D)
    return lpr + int(math.log2(32 // lpr)) + 8 + (kd_chunks(S) + 4 * G - 1) // (4 * G) + 3 + 2 + G + 1


def keydiff_ref64(k: torch.Tensor) -> torch.Tensor:
    """anchor = mean_s k_s / max(||k_s||, 1e-12); score_s = -(k_s . a) / (max(||k_s||, 1e-8) max(||a||, 1e-8)),
    in float64 on k's device, one batch at a time."""
    out = []
    for b in range(k.shape[0]):
        kk = k[b].double()
        n = kk.norm(dim=-1)
        a = (kk / n.clamp_min(1e-12)[..., None]).mean(1)
        an = a.norm(dim=-1).clamp_min(1e-8)
        out.append(-(kk @ a[..., None])[..., 0] / (n.clamp_min(1e-8) * an[:, None]))
    return torch.stack(out)


def keydiff_error_bound(k: torch.Tensor, chain: int) -> torch.Tensor:
    """E_s of the module docstring, [B, H, S] float64. Keys that are not finite, or whose fp32 sum of squares is not,
    weigh nothing in the kernel's anchor (their rows are NaN, or their 1 / ||k|| is 0) and are left out."""
    D = k.shape[-1]
    out = []
    for b in range(k.shape[0]):
        kf = k[b].float()
        live = torch.isfinite((kf * kf).sum(-1))
        kk = torch.where(live[..., None], k[b].double(), 0.0)
        n = kk.norm(dim=-1)
        kh = kk / n.clamp_min(1e-12)[..., None]
        a = kh.mean(1)
        an = a.norm(dim=-1).clamp_min(1e-8)
        m = kh.abs().mean(1)
        den = n.clamp_min(1e-8) * an[:, None]
        ref = (kk @ a[..., None])[..., 0].abs() / den
        e_dot = (kk.abs() @ a.abs()[..., None])[..., 0] / den
        e_anchor = (kk.abs() @ m[..., None])[..., 0] / den + ref * ((a.abs() * m).sum(-1) / an ** 2)[:, None]
        out.append(U32 * ((D + 8) * e_dot + (chain + 16) * e_anchor + 24 * ref))
    return torch.stack(out)


def assert_keydiff_vs_ref(got, ref, E, what: str, bias: bool = True, e_factor: float = 1.0) -> dict:
    """The bar of the module docstring: NaN where ref is NaN; elsewhere <= 1 ulp of round16(ref) or within
    ulp16(got) / 2 + e_factor E_s of ref; no row bias. Returns the measured statistics."""
    dtype = got.dtype
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(got), nan), f"{what}: NaN scores differ from the reference's"
    r16 = torch.where(nan, 0.0, ref).to(dtype)
    g = torch.where(nan, torch.zeros_like(got), got)
    d = ulp16_diff(g, r16)
    ok = d <= 1
    e_arm = (g.double() - torch.where(nan, 0.0, ref)).abs() <= 0.5 * ulp16(g) + e_factor * E
    bad = ~(ok | e_arm)
    if bad.any():
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} scores beyond both arms, first at {i}: got {float(got[tuple(i)])} "
                             f"ref {float(ref[tuple(i)])} E {float(E[tuple(i)]):.3e} ({int(d[tuple(i)])} ulp)")
    only_e = ~ok
    # positions the E arm decides enter the 1-ulp and bias bars at round16(ref); NaN rows are left out (0)
    stats = assert_vs_ref64(torch.where(only_e, r16, g), torch.where(nan, 0.0, ref), torch.zeros(ref.shape[-1], dtype=torch.bool),
                            what, bias=bias)
    fin = ~nan
    stats["e_only"] = float(only_e[fin].float().mean()) if fin.any() else 0.0
    stats["max_e"] = float(E[fin].max()) if fin.any() else 0.0
    print(f"[measured] {what}: share decided by the E arm {stats['e_only']:.2e}, max E_s {stats['max_e']:.2e}")
    return stats


def assert_e_small(E, ref, what: str):
    """max E_s of every (b, h) row <= E_SCALE_FRACTION of its largest |score|"""
    fin = torch.isfinite(ref)
    scale = torch.where(fin, ref.abs(), 0.0).amax(-1)
    worst = torch.where(fin, E, 0.0).amax(-1)
    ok = worst <= E_SCALE_FRACTION * scale
    assert ok.all(), f"{what}: E_s up to {float((worst / scale.clamp_min(1e-300)).max()):.2e} of the row's score scale"


def rope_inv_freq(kind: str, D: int, seed: int = 0) -> torch.Tensor:
    """fp32 [D / 2] as a model computes it"""
    exps = torch.arange(0, D, 2, dtype=torch.int64).float() / D
    if kind.startswith("theta"):
        return 1.0 / (float(kind[5:]) ** exps)
    if kind == "yarn_like":  # the low frequencies interpolated by up to 8x, the high ones kept
        return 1.0 / (500000.0 ** exps) / torch.linspace(1.0, 8.0, D // 2)
    # random_first_one: log-uniform over [1e-7, 1], descending, the first exactly 1
    g = torch.Generator().manual_seed(seed)
    inv = torch.exp2(-torch.rand(D // 2, generator=g) * 23.25).sort(descending=True).values
    inv[0] = 1.0
    return inv


def scores64(k, q, w, normalize=True, rows=64):
    """FinchPress: float64 [B, H, S - w] context scores, window rows in blocks."""
    B, H, S, D = k.shape
    G = q.shape[1] // H
    kk = k.double()
    qq = q.double().reshape(B, H, G, w, D)
    col = torch.zeros(B, H, S - w, dtype=torch.float64, device=k.device)
    pos = torch.arange(S, device=k.device)
    for i0 in range(0, w, rows):
        i1 = min(w, i0 + rows)
        y = torch.einsum("bhgid,bhsd->bhgis", qq[:, :, :, i0:i1], kk) / math.sqrt(D)
        rpos = torch.arange(S - w + i0, S - w + i1, device=k.device)
        y.masked_fill_(pos[None, :] > rpos[:, None], float("-inf"))
        p = torch.softmax(y, dim=-1)[..., : S - w]
        if normalize:
            p = p * rpos.double()[:, None]
        col += p.sum(dim=(2, 3))
    return col / (G * w)


def assert_scores(got, k, q, w, normalize, what):
    """FinchPress's bar (tests/test_gpu_finch.py): every context score within 1 ulp of the float64 value, the window
    holding round(max + 1)."""
    S = k.shape[2]
    ref = scores64(k, q, w, normalize)
    ctx = got[..., : S - w].double()
    err = (ctx - ref).abs()
    bound = ulp_at(ref, got.dtype)
    bad = err > bound
    assert not bad.any(), f"{what}: {int(bad.sum())} scores beyond 1 ulp, worst {float((err / bound).max())} ulp"
    sentinel = (got[..., : S - w].float().max() + 1).to(got.dtype)
    assert (got[..., S - w:] == sentinel).all(), f"{what}: window sentinel"


# ---------------------------------------------------------------------------------------------------
# the exact selection contract (tests/test_gpu_select_compact_sweep.py, tests/test_gpu_chunked_select_sweep.py)
# ---------------------------------------------------------------------------------------------------
INF_BITS = {torch.bfloat16: 0x7F80, torch.float16: 0x7C00}
# kTile / kTileThreads of common.cuh (the select sweep's CPU test checks them against the source)
TILE = 256
TILE_THREADS = 256


def copy_edges(u: int):
    """copy_rows_kv<u> copies count·nvec vectors in steps of TILE_THREADS·u, two steps per loop iteration"""
    step = TILE_THREADS * u
    return (step, 2 * step)


def edge_counts(nvec: int, u: int):
    """kept counts of one tile whose count·nvec is the last multiple of nvec below, the first at or above, and the
    first above each copy edge, where a tile can hold them; and 1 and a full tile"""
    out = {1, TILE}
    for e in copy_edges(u):
        out |= {(e - 1) // nvec, -(-e // nvec), e // nvec + 1}
    return sorted(c for c in out if 1 <= c <= TILE)


def key16(bits: torch.Tensor, dtype) -> torch.Tensor:
    """`ordered_key16` restated on int64, only to place n_kept at the kernels' bin edges (never to judge a result)"""
    b = bits.long() & 0xFFFF
    nan = (b & 0x7FFF) > INF_BITS[dtype]
    b = torch.where(b == 0x8000, 0, b)
    key = torch.where(b >= 0x8000, (~b) & 0xFFFF, b | 0x8000)
    return torch.where(nan, 0xFFFF, key)


def oracle_key(scores: torch.Tensor) -> torch.Tensor:
    """The ranking key of `O.select_lowest_index_ties`: float value, -0 == +0, every NaN above +inf"""
    s = scores.float()
    s = torch.where(s == 0, torch.zeros_like(s), s)
    bits = s.contiguous().view(torch.int32).to(torch.int64)
    key = torch.where(bits < 0, -(bits & 0x7FFFFFFF), bits)
    return torch.where(torch.isnan(s), torch.full_like(key, 2 ** 40), key)


def canonical_order(scores: torch.Tensor) -> torch.Tensor:
    """positions of every row by descending score, equal scores in ascending position order"""
    return torch.sort(oracle_key(scores), dim=-1, descending=True, stable=True).indices


def canonical(order: torch.Tensor, n: int) -> torch.Tensor:
    return torch.sort(order[..., :n], dim=-1).values


def chunk_orders(scores: torch.Tensor, L: int):
    """The canonical order of each full chunk of L positions ([..., n_full, L], None without one) and of the short last
    chunk ([..., S % L], None without one), positions relative to the chunk's start."""
    S = scores.shape[-1]
    n_full = S // L
    full = canonical_order(scores[..., : n_full * L].unflatten(-1, (n_full, L))) if n_full else None
    tail = canonical_order(scores[..., n_full * L:]) if S % L else None
    return full, tail


def chunked_from_orders(orders, L: int, chunk_kept: int, tail_kept: int) -> torch.Tensor:
    """The chunked selection: chunk c holds positions [c L, min(S, (c + 1) L)); each full chunk keeps the canonical
    top chunk_kept of its own scores, the short last chunk its top tail_kept, each ascending and offset by the chunk's
    start, the chunks in order. int64 [..., n_full chunk_kept + tail_kept]."""
    full, tail = orders
    parts = []
    if full is not None:
        n_full = full.shape[-2]
        kept = canonical(full, chunk_kept) + torch.arange(0, n_full * L, L, device=full.device)[:, None]
        parts.append(kept.flatten(-2))
    if tail is not None:
        n_full = 0 if full is None else full.shape[-2]
        parts.append(canonical(tail, tail_kept) + n_full * L)
    return torch.cat(parts, dim=-1)


def chunked_canonical(scores: torch.Tensor, L: int, chunk_kept: int, tail_kept: int) -> torch.Tensor:
    return chunked_from_orders(chunk_orders(scores, L), L, chunk_kept, tail_kept)


def chunked_oracle(scores: torch.Tensor, L: int, chunk_kept: int, tail_kept: int) -> torch.Tensor:
    """`O.select_lowest_index_ties` applied chunk by chunk on the CPU (slow: one call per chunk)"""
    S = scores.shape[-1]
    s = scores.cpu()
    parts = []
    for lo in range(0, S, L):
        hi = min(S, lo + L)
        parts.append(O.select_lowest_index_ties(s[..., lo:hi], chunk_kept if hi - lo == L else tail_kept) + lo)
    return torch.cat(parts, dim=-1)


def all_patterns(dtype) -> torch.Tensor:
    return torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(dtype)


def key_space_n_kept(keys: torch.Tensor, dtype):
    """n_kept at every high-byte boundary c_b = #{key >> 8 >= b} and c_b +- 1, at every low-byte boundary of the bins
    of NaN, +inf, -inf, +-0 and the subnormals, and 1, S - 1, S"""
    S = keys.numel()
    hi = keys >> 8
    ns = {1, S - 1, S}
    for b in range(256):
        c = int((hi >= b).sum())
        ns |= {c - 1, c, c + 1}
    inf = INF_BITS[dtype]
    special = torch.tensor([0xFFFF, 0x8000 | inf, (~(0x8000 | inf)) & 0xFFFF], dtype=torch.int64)  # NaN, +inf, -inf
    sub = torch.arange(1, 1 << (10 if dtype == torch.float16 else 7))
    bins = set((special >> 8).tolist()) | set((key16(torch.cat([sub, sub | 0x8000, torch.tensor([0])]), dtype) >> 8).tolist())
    for b in bins:
        for lo in range(256):
            ns.add(int((keys >= (b << 8 | lo)).sum()))
    return sorted(n for n in ns if 1 <= n <= S)


def _pattern_keys(dtype):
    pats = all_patterns(dtype).view(torch.int16)
    return pats, key16(pats, dtype)


def threshold_patterns(kind: str, dtype) -> torch.Tensor:
    """the bit patterns of one threshold key (several for NaN and zero)"""
    pats, keys = _pattern_keys(dtype)
    inf = INF_BITS[dtype]
    if kind == "neg_inf":
        t = keys[pats.long() == (inf | 0x8000) - 65536]
    elif kind == "most_negative":
        t = keys[pats.long() == ((inf - 1) | 0x8000) - 65536]
    elif kind == "nan":
        t = torch.tensor([0xFFFF])
    elif kind == "zero_mixed_sign":
        t = torch.tensor([0x8000])
    elif kind == "key_lo00":  # a negative value whose key ends in 0x00
        t = torch.tensor([0x4000])
    else:  # key_loff: a positive value whose key ends in 0xFF
        t = torch.tensor([0xBFFF])
    return pats[keys == int(t[0])]


def rand_bits(shape, gen, dtype) -> torch.Tensor:
    return torch.randint(-32768, 32768, tuple(shape), generator=gen, device=DEV, dtype=torch.int16).view(dtype)


def mixed_scores(shape, dtype, gen) -> torch.Tensor:
    """random bit patterns, half of them replaced by a few tied values: +-0, -inf, two NaN payloads, 1, -1"""
    x = rand_bits(shape, gen, dtype)
    pool = torch.tensor([0, -0.0, float("-inf"), 1.0, -1.0], dtype=dtype, device=DEV).view(torch.int16)
    pool = torch.cat([pool, torch.tensor([INF_BITS[dtype] + 1, -1], dtype=torch.int16, device=DEV)]).view(dtype)
    pick = torch.randint(0, pool.numel(), tuple(shape), generator=gen, device=DEV)
    tied = torch.rand(tuple(shape), generator=gen, device=DEV) < 0.5
    return torch.where(tied, pool[pick], x)


def kv_for(B, H, S, D, dtype, gen):
    """K, V of random bit patterns (NaN payloads included), and finite keys for the re-rotating call"""
    return (rand_bits((B, H, S, D), gen, dtype), rand_bits((B, H, S, D), gen, dtype),
            torch.randn(B, H, S, D, generator=gen, device=DEV).to(dtype))


def _poison(*nbytes) -> set:
    """Allocates blocks of these sizes in this order, fills them with 0xFF and frees them: the caching allocator hands
    the same blocks to allocations of the same sizes in the same order. Returns their addresses."""
    blocks = [torch.empty(n, dtype=torch.uint8, device=DEV) for n in nbytes if n > 0]
    for b in blocks:
        b.fill_(0xFF)
    return {b.data_ptr() for b in blocks}


def _landed(ptrs: set, *outs):
    for o in outs:
        if o is not None and o.numel() > 0:
            assert o.data_ptr() in ptrs, "an output did not land on a poisoned block"


def _score_copy_bytes(scores, dtype) -> int:
    """bytes of the copy the binding makes of scores it cannot pass as they are (other dtype, or S not unit-stride)"""
    if scores.dtype != dtype:
        return scores.numel() * 2 + (scores.numel() * 2 if scores.stride(2) != 1 else 0)
    return scores.numel() * 2 if scores.stride(2) != 1 else 0


def _kv_out_bytes(k, n):
    B, H, _, D = k.shape
    return [B * H * n * D * 2] * 2 + [B * H * n * 4]


def assert_idx(idx, want, what):
    assert idx.dtype == torch.int32, f"{what}: idx is {idx.dtype}"
    if not torch.equal(idx.long(), want):
        bad = (idx.long() != want).nonzero()
        i = bad[0].tolist()
        raise AssertionError(f"{what}: {bad.shape[0]} of {want.numel()} kept positions differ from the canonical "
                             f"selection, first at {i}: got {int(idx[tuple(i)])}, want {int(want[tuple(i)])}")


def assert_gather(out, x, want, what):
    assert torch.equal(_bits(out), _bits(_gather(x, want))), f"{what}: not a bitwise gather"


def rerotation_admissible(k: torch.Tensor, idx: torch.Tensor, inv_freq: torch.Tensor) -> torch.Tensor:
    """[4, B, H, n, D]: k[idx] rotated by (j - idx_j) * inv_freq with every admissible (cos16, sin16) pair."""
    dtype, D = k.dtype, k.shape[-1]
    g = _gather(k, idx)
    delta = torch.arange(idx.shape[-1], device=k.device, dtype=torch.float32) - idx.float()  # exact below 2^24
    ang = (delta[..., None] * inv_freq.to(k.device, torch.float32)).double()  # one fp32 multiply, as the kernel's
    cands = []
    for f in (torch.cos, torch.sin):
        x = f(ang)
        tol = 2 * _ulp32(x * (1 + 2.0 ** -20))  # sincosf: 2 ulp, in the larger binade at a binade edge
        cands.append([((x - tol).float().to(dtype)), ((x + tol).float().to(dtype))])
    out = []
    for c in cands[0]:
        for s in cands[1]:
            out.append(g * torch.cat((c, c), -1) + O.rotate_half(g) * torch.cat((s, s), -1))
    return torch.stack(out)


def assert_rerotated(k, v, scores, n, inv_freq, out, what: str) -> int:
    """canonical idx, exact V' gather, every K' element one of the admissible results; returns the count of elements
    with more than one admissible result."""
    k_out, v_out, idx = out
    assert torch.equal(idx.long().cpu(), O.select_lowest_index_ties(scores.cpu(), n)), f"{what}: not the canonical selection"
    assert _same(v_out, _gather(v, idx)), f"{what}: V' is not an exact gather"
    adm = _bits(rerotation_admissible(k, idx, inv_freq))
    hit = (adm == _bits(k_out)[None]).any(0)
    if not hit.all():
        i = (~hit).nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int((~hit).sum())} of {hit.numel()} K' elements not admissible, first at {i}: "
                             f"got {float(k_out[tuple(i)])}, admissible {adm[(slice(None), *i)].view(k.dtype).tolist()}")
    return int((adm != adm[:1]).any(0).sum())
