/*
 * kvpress_b200.h — C ABI of the H100-native (sm_90a) fused KV-cache compression path.
 *
 * The reference (NVIDIA/kvpress, pure Python/PyTorch) has no FFI: its hot path is the ATen
 * sequence inside ScorerPress.compress (kvpress/presses/scorer_press.py:76-102):
 *     scores = self.score(...)                     (:90)   per-scorer, see below
 *     n_kept = int(k_len * (1 - ratio))            (:93-94) computed by the HOST and passed in
 *     indices = scores.topk(n_kept).indices        (:95)
 *     keys/values.gather(2, indices).contiguous()  (:99-100)
 * Every entry point below replaces that sequence (or its score() part) for one scorer:
 *     kvp_knorm_*              <- kvpress/presses/knorm_press.py:29-38
 *     kvp_streaming_*          <- kvpress/presses/streaming_llm_press.py:38-54
 *     kvp_snapkv_*             <- kvpress/presses/snapkv_press.py:41-105
 *     kvp_expected_attention_* <- kvpress/presses/expected_attention_press.py:126-165
 *     kvp_keydiff_*            <- kvpress/presses/keydiff_press.py:36-46
 *     kvp_criticalkv_*         <- kvpress/presses/criticalkv_press.py:57-92 (on the wrapped press's scores)
 *     kvp_observed_attention_* <- kvpress/presses/observed_attention_press.py (H2O; from Q and K, no eager weights)
 *     kvp_non_causal_attention_* <- kvpress/presses/non_causal_attention_press.py (Compactor's attention half)
 *     kvp_lagkv_*              <- kvpress/presses/lagkv_press.py (lag-relative K / V statistics, from K and V only)
 *     kvp_cur_*                <- kvpress/presses/cur_press.py (approximate K / V leverage scores, from K and V only)
 *     kvp_merging_*            <- kvpress/presses/merging_press.py (evicted values folded into their nearest kept row)
 *     kvp_think_prune          <- kvpress/presses/think_press.py (key channels zeroed in place; no positions removed)
 *     kvp_cam_compress         <- kvpress/presses/cam_press.py (evicted values merged into the kept rows after them)
 *     kvp_kvzap_*              <- kvpress/presses/kvzap_press.py (a surrogate model of the hidden states)
 *     kvp_threshold_evict      <- kvpress/presses/dms_press.py (the positions whose score is below a threshold)
 *     kvp_scores_compress      <- scorer_press.py:93-100 for an arbitrary score tensor
 *                                 (what wrapper presses / user ScorerPress subclasses need)
 *
 * Conventions
 *   - All pointers are DEVICE pointers unless a name ends in _host. Nothing here is a torch type.
 *   - K, V: [B, Hkv, S, D], 16-bit floats (bf16 or fp16), innermost dim contiguous, outer dims
 *     arbitrary element strides (kvp_problem.k_stride / v_stride), 16-byte aligned rows.
 *   - Outputs K_out, V_out: contiguous [B, Hkv, n_kept, D]; rows in ASCENDING POSITION order
 *     (the reference emits score-descending order; attention is permutation invariant over
 *     (K,V) rows — see DESIGN.md "row order").
 *   - idx_out (nullable): int32 [B, Hkv, n_kept], the kept positions, ascending.
 *   - scores_out (nullable): [B, Hkv, S] in the K dtype, same values the reference's score()
 *     returns (including the max+1 sentinel on forced-keep positions).
 *   - Selection rule: the n_kept largest scores per (b, h) row; ties at the threshold are
 *     resolved towards the LOWEST position (deterministic; torch.topk leaves it unspecified).
 *   - Caller owns all memory (outputs + workspace of kvp_workspace_bytes()). The library
 *     allocates no device memory and never synchronises the stream (kvp_workspace_check excepted).
 *     Every kernel runs on the caller's stream. The only process-wide state is write-once caches of
 *     per-device properties: SM count, occupancy and function attributes. Calls are re-entrant per
 *     (stream, workspace); every call is CUDA-graph capturable.
 *   - Return value: KVP_OK (0) or a negative kvp_status. No exceptions cross this boundary.
 */
#ifndef KVPRESS_B200_H
#define KVPRESS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KVP_ABI_VERSION 1

typedef void* kvp_stream_t; /* a cudaStream_t */

typedef enum kvp_status {
    KVP_OK = 0,
    KVP_ERR_NULL_POINTER = -1,
    KVP_ERR_UNSUPPORTED_SHAPE = -2,
    KVP_ERR_UNSUPPORTED_DTYPE = -3,
    KVP_ERR_BAD_STRIDE = -4,
    KVP_ERR_WORKSPACE_TOO_SMALL = -5,
    KVP_ERR_CUDA = -6,
    KVP_ERR_BAD_ARGUMENT = -7,
    KVP_ERR_KERNEL_TIMEOUT = -8 /* a kernel abandoned a bounded wait: outputs invalid (library bug) */
} kvp_status;

typedef enum kvp_dtype { KVP_BF16 = 0, KVP_F16 = 1 } kvp_dtype;

typedef enum kvp_scorer {
    KVP_SCORER_GENERIC = 0, /* scores supplied by the caller            */
    KVP_SCORER_KNORM = 1,
    KVP_SCORER_STREAMING = 2,
    KVP_SCORER_SNAPKV = 3,
    KVP_SCORER_EXPECTED_ATTENTION = 4,
    KVP_SCORER_KEYDIFF = 5,
    KVP_SCORER_CRITICALKV = 6,
    KVP_SCORER_OBSERVED_ATTENTION = 7,
    KVP_SCORER_NON_CAUSAL_ATTENTION = 8,
    KVP_SCORER_LAGKV = 9,
    /* 10, 12 and 15 are not assigned: kvp_launches_per_compress answers KVP_ERR_BAD_ARGUMENT for them, as for any
     * unknown id */
    KVP_SCORER_CUR = 11,
    KVP_SCORER_MERGING = 13, /* kvp_merging_*: the selection of the caller's scores, then the merge */
    KVP_SCORER_THINK = 14,   /* kvp_think_prune: key channels, not positions */
    KVP_SCORER_FINCH = 16,   /* kvp_finch_*, kvp_scores_compress_chunked */
    KVP_SCORER_CAM = 17,     /* kvp_cam_compress */
    KVP_SCORER_KVZAP = 18    /* kvp_kvzap_* */
} kvp_scorer;

/* One ScorerPress.compress call on one layer's cache. */
typedef struct kvp_problem {
    int32_t B;      /* batch                                                         */
    int32_t Hkv;    /* key/value heads                                               */
    int32_t Hq;     /* query heads (multiple of Hkv; = Hkv when the scorer has no Q) */
    int32_t S;      /* k_len, cached positions                                       */
    int32_t D;      /* head_dim (multiple of 8, <= 256)                              */
    int32_t n_kept; /* int(S * (1 - compression_ratio)), computed by the host        */
    int32_t dtype;  /* kvp_dtype of K, V, scores, Q, mu, cov                         */
    int32_t reserved;
    int64_t k_stride[3]; /* element strides of K for (b, h, s); stride of d is 1 */
    int64_t v_stride[3]; /* element strides of V for (b, h, s)                   */
} kvp_problem;

/* ---- library info ---------------------------------------------------------------------- */
int kvp_abi_version(void);
const char* kvp_status_string(int status);
/* Last CUDA error string recorded on this host thread by a failed call (never NULL). */
const char* kvp_last_cuda_error(void);

/* Bytes of scratch a *_compress / *_score call of this scorer needs (256-byte aligned), whatever its other arguments:
 * every SnapKV window, ObservedAttention n_q, CUR window / rank, ... the call accepts. */
int kvp_workspace_bytes(const kvp_problem* p, int scorer, size_t* bytes_out);

/* Debugging aid. The persistent select / compact kernels wait on each other with BOUNDED spins; a wait that
 * expires raises a flag in the workspace instead of trapping the CUDA context. This call synchronises
 * `stream`, reads the flag of the last call that used `workspace` and returns KVP_OK or
 * KVP_ERR_KERNEL_TIMEOUT. Never needed for correct operation. */
int kvp_workspace_check(const kvp_problem* p, int scorer, const void* workspace, size_t workspace_bytes,
                        kvp_stream_t stream);

/* Number of kernel launches (incl. memset nodes) one *_compress call enqueues; bench.py
 * reports it as gpu_launches. */
int kvp_launches_per_compress(const kvp_problem* p, int scorer, int* launches_out);

/* ---- KnormPress: score = -||k||_2 (fp32 accumulate, one rounding to the K dtype) ------- */
int kvp_knorm_score(const kvp_problem* p, const void* K, void* scores_out, kvp_stream_t stream);
int kvp_knorm_compress(const kvp_problem* p, const void* K, const void* V, void* K_out,
                       void* V_out, int32_t* idx_out, void* scores_out, void* workspace,
                       size_t workspace_bytes, kvp_stream_t stream);

/* ---- StreamingLLMPress: keep [0, n_sink) and the most recent positions ------------------ */
int kvp_streaming_score(const kvp_problem* p, int32_t n_sink, void* scores_out,
                        kvp_stream_t stream);
int kvp_streaming_compress(const kvp_problem* p, int32_t n_sink, const void* K, const void* V,
                           void* K_out, void* V_out, int32_t* idx_out, kvp_stream_t stream);

/* ---- SnapKVPress -------------------------------------------------------------------------
 * q_window: RoPE'd queries of the last `window` positions, contiguous [B, Hq, window, D]
 * (snapkv_press.py:53-58 — the 64-row q_proj GEMM + RoPE is the caller's prologue).
 * Scores: softmax over all S keys (causal inside the window) of q·k/sqrt(D), mean over the
 * window queries, avg_pool1d(kernel_size, pad=kernel_size/2, stride 1, divisor kernel_size),
 * mean over the Hq/Hkv group; the last `window` positions are always kept. */
int kvp_snapkv_score(const kvp_problem* p, const void* K, const void* q_window, int32_t window,
                     int32_t kernel_size, void* scores_out, void* workspace,
                     size_t workspace_bytes, kvp_stream_t stream);
int kvp_snapkv_compress(const kvp_problem* p, const void* K, const void* V,
                        const void* q_window, int32_t window, int32_t kernel_size, void* K_out,
                        void* V_out, int32_t* idx_out, void* scores_out, void* workspace,
                        size_t workspace_bytes, kvp_stream_t stream);

/* ---- ExpectedAttentionPress --------------------------------------------------------------
 * mu: [B, Hq, D], cov: [B, Hq, D, D] (nullable = use_covariance False), both already rotated
 * by the average RoPE matrix (expected_attention_press.py:62-124 — the query-statistics
 * prologue stays with the caller). Scores over positions [n_sink, S):
 *   softmax_s( mu·k/sqrt(D) + k^T cov k / (2 D) ), mean over the group, (+eps) * ||v||_2 when
 *   use_vnorm; the first n_sink positions are always kept. */
int kvp_expected_attention_score(const kvp_problem* p, const void* K, const void* V,
                                 const void* mu, const void* cov, float epsilon, int32_t n_sink,
                                 int32_t use_vnorm, void* scores_out, void* workspace,
                                 size_t workspace_bytes, kvp_stream_t stream);
int kvp_expected_attention_compress(const kvp_problem* p, const void* K, const void* V,
                                    const void* mu, const void* cov, float epsilon,
                                    int32_t n_sink, int32_t use_vnorm, void* K_out, void* V_out,
                                    int32_t* idx_out, void* scores_out, void* workspace,
                                    size_t workspace_bytes, kvp_stream_t stream);

/* ---- generic: top-k + compaction of caller-supplied scores ------------------------------
 * scores: [B, Hkv, S] in the K dtype with element strides score_stride (b, h; s contiguous). */
int kvp_scores_compress(const kvp_problem* p, const void* scores, const int64_t* score_stride,
                        const void* K, const void* V, void* K_out, void* V_out,
                        int32_t* idx_out, void* workspace, size_t workspace_bytes,
                        kvp_stream_t stream);

/* ---- KeyDiffPress (kvpress/presses/keydiff_press.py:36-46): score = -cos(k, anchor), anchor = mean over
 * positions of k / ||k||; fp32 evaluation, one rounding to the K dtype. Two streaming passes over K. */
int kvp_keydiff_score(const kvp_problem* p, const void* K, void* scores_out, void* workspace,
                      size_t workspace_bytes, kvp_stream_t stream);
int kvp_keydiff_compress(const kvp_problem* p, const void* K, const void* V, void* K_out, void* V_out,
                         int32_t* idx_out, void* scores_out, void* workspace, size_t workspace_bytes,
                         kvp_stream_t stream);

/* ---- CriticalKVPress (kvpress/presses/criticalkv_press.py:57-92) on the scores of the press it wraps ----------------
 * base_scores: [B, Hkv, S] in the K dtype with element strides score_stride (b, h; s contiguous), 2-byte aligned.
 * wo: o_proj.weight, [hidden, Hq*D] rows with row stride wo_stride (a multiple of 8, >= Hq*D), 16-byte aligned.
 * With G = Hq / Hkv and the query heads h = j G + g of kv head j:
 *   norm[b,j,s]  = (1/G) sum_g sum_{n < hidden} | sum_d V[b,j,s,d] wo[n, h D + d] |
 *   score[b,j,s] = (base_scores[b,j,s] + epsilon) * norm[b,j,s]     (fp32, one rounding to the K dtype)
 * then the n_first positions of every row with the largest base score (ties to the lowest positions) get the dtype's
 * largest finite value; the host computes n_first = int((1 - ratio) * S * first_stage_ratio). head_dim 64 or 128
 * (else KVP_ERR_UNSUPPORTED_SHAPE), any G and hidden. n_first is at most S for the score call and at most n_kept for
 * the compress call, which then keeps the n_kept best final scores (scores_out nullable). K is only gathered. */
int kvp_criticalkv_score(const kvp_problem* p, const void* V, const void* base_scores, const int64_t* score_stride,
                         const void* wo, int32_t hidden, int64_t wo_stride, float epsilon, int32_t n_first,
                         void* scores_out, void* workspace, size_t workspace_bytes, kvp_stream_t stream);
int kvp_criticalkv_compress(const kvp_problem* p, const void* K, const void* V, const void* base_scores,
                            const int64_t* score_stride, const void* wo, int32_t hidden, int64_t wo_stride,
                            float epsilon, int32_t n_first, void* K_out, void* V_out, int32_t* idx_out,
                            void* scores_out, void* workspace, size_t workspace_bytes, kvp_stream_t stream);

/* ---- ObservedAttentionPress (kvpress/presses/observed_attention_press.py, the H2O score) -------------------------------
 * q: the RoPE'd queries of the current forward, contiguous [B, Hq, n_q, D], 16-byte aligned; row i is at position
 * p_i = S - n_q + i (1 <= n_q <= S: n_q = S in prefill, the current step's rows under DecodingPress). With G = Hq / Hkv
 * and the query heads h = j G + g of kv head j:
 *   y[b,h,i,s]   = scaling * q[b,h,i] . K[b,j,s] for s <= p_i, else -inf     (scaling: the attention's module.scaling)
 *   P[b,h,i,s]   = softmax over s of y                                      (exact normaliser over the whole row)
 *   score[b,j,s] = (1/G) sum_g sum_i P[b,h,i,s] / c(S - s)                  (fp32, one rounding to the K dtype)
 * where c(n) is n rounded to the K dtype, as the reference divides by torch.arange(S, 0, -1) in the attention dtype:
 * counts above 256 round in bf16, and in fp16 counts of 65520 and above are inf, so those first positions score
 * exactly 0. No position is forced. head_dim 64 or 128 and 1 <= G <= 8, else KVP_ERR_UNSUPPORTED_SHAPE.
 * Check order (the first failure is returned): validate the problem -> n_kept == 0 returns KVP_OK (compress) ->
 * K / V / K_out / V_out null and alignment (compress) -> q null / alignment (and K, scores_out for the score call) ->
 * 1 <= n_q <= S, else KVP_ERR_BAD_ARGUMENT -> scaling finite and > 0, else KVP_ERR_BAD_ARGUMENT -> workspace.
 * kvp_workspace_bytes sizes the workspace for n_q = S. The compress call keeps the n_kept best scores (scores_out
 * nullable). Memory beyond the workspace: none; the [B, Hq, n_q, S] weights are never formed. */
int kvp_observed_attention_score(const kvp_problem* p, const void* K, const void* q, int32_t n_q, float scaling,
                                 void* scores_out, void* workspace, size_t workspace_bytes, kvp_stream_t stream);
int kvp_observed_attention_compress(const kvp_problem* p, const void* K, const void* V, const void* q, int32_t n_q,
                                    float scaling, void* K_out, void* V_out, int32_t* idx_out, void* scores_out,
                                    void* workspace, size_t workspace_bytes, kvp_stream_t stream);

/* ---- NonCausalAttnPress (kvpress/presses/non_causal_attention_press.py, the attention half of Compactor) -------------
 * Prefill only. q: the RoPE'd queries of all S positions, contiguous [B, Hq, S, D], 16-byte aligned. With G = Hq / Hkv,
 * the query heads h = j G + g of kv head j, cs = chunk_size and the chunks [c cs, (c+1) cs) of positions:
 *   y[b,h,i,s]   = q[b,h,i] . K[b,j,s]  for i, s in the same chunk        (NO 1/sqrt(D) scaling)
 *   A[b,h,s]     = sum_i softmax over the chunk's keys of y[b,h,i,:] at s   (non-causal)
 *   x[b,j,s]     = (1/G) sum_g A[b,h,s] * ||V[b,j,s]||_2
 *   pooled       = avg_pool1d(x, 3, padding 1, stride 1)                     (zeros outside [0, S), always / 3)
 *   score        = (pooled - mean) / max(std, 1e-6)                          (fp32 evaluation, ONE rounding to the K dtype)
 * mean and the unbiased std run over ALL B*Hkv*S entries, so the rows of a batch are coupled, and B*Hkv*S = 1 gives
 * NaN, as torch's std. Padding of the last chunk (S not a multiple of cs; pad = ceil(S/cs) cs - S), as the reference:
 * the pad padded keys are NOT masked, every valid query row of the last chunk sees them at logit 0 (the reference's
 * -1e-9, to fp32 resolution); each of the pad padded query rows adds a uniform 1/cs to every valid key of that chunk.
 * The reference rounds the logits and ||v|| to the cache dtype and returns fp32 z; here the formula is evaluated in fp32
 * from the 16-bit inputs and z is rounded once. Selection keeps the n_kept largest rounded z (ties to the lowest
 * positions), exactly what scores_out holds. head_dim 64 or 128, chunk_size 128 or 256 and 1 <= G <= 8, else
 * KVP_ERR_UNSUPPORTED_SHAPE.
 * Check order (the first failure is returned): validate the problem -> n_kept == 0 returns KVP_OK (compress) ->
 * K / V / K_out / V_out null and alignment (compress) -> q null / alignment (and K, V, scores_out for the score call) ->
 * chunk_size >= 1, else KVP_ERR_BAD_ARGUMENT -> shape instantiated, else KVP_ERR_UNSUPPORTED_SHAPE -> workspace.
 * The compress call keeps the n_kept best scores (scores_out nullable). Memory beyond the workspace: none; no cs x cs
 * tensor is formed. */
int kvp_non_causal_attention_score(const kvp_problem* p, const void* K, const void* V, const void* q,
                                   int32_t chunk_size, void* scores_out, void* workspace, size_t workspace_bytes,
                                   kvp_stream_t stream);
int kvp_non_causal_attention_compress(const kvp_problem* p, const void* K, const void* V, const void* q,
                                      int32_t chunk_size, void* K_out, void* V_out, int32_t* idx_out,
                                      void* scores_out, void* workspace, size_t workspace_bytes,
                                      kvp_stream_t stream);

/* ---- LagKVPress (kvpress/presses/lagkv_press.py, https://arxiv.org/abs/2504.04704) ----------------------------------
 * Reads K and V only. Per row (b, kv head j), with S positions and L = lag_size:
 *   - Short cache, S < n_sink + 2L. Position s < n_sink scores 1. Position s >= n_sink scores
 *     fp32(s - n_sink) / fp32(S - n_sink), rounded once to the cache dtype (the reference's float32 arange / n).
 *   - Otherwise P = (S - n_sink) // L, partition c covers [n_sink + cL, n_sink + (c+1)L), and partitions
 *     c = 0 ... P-2 are scored, each against partition c+1. The sinks, partition P-1 and the remainder score 1.
 *   - Within a scored partition, per channel d: lo_d / hi_d = min / max over the reference partition's L rows,
 *     x = (k - lo) / (hi - lo) with IEEE rules (x/0 = +-inf, 0/0 = NaN), sigma_k = unbiased std of x over d
 *     (divisor D - 1), a_k = softmax of sigma_k over the L rows; sigma_v and a_v likewise from V;
 *     c = (a_k + a_v) / 2.
 *   - cross_scoring != 0: the score is c rounded once. Otherwise it is fp32(r) / fp32(L) rounded once, with the rank
 *     r(s) = #{t : c(t) < c(s)} + #{t < s : c(t) = c(s)} over the partition; NaN compares above every number and equal
 *     to NaN (torch.sort(stable=True)).
 * A constant channel of a reference partition, in K or V (a zeroed channel, or any partition when L = 1), makes every c
 * of the partition it scores NaN: NaN cross scores and ranks in position order, as in the reference. So does a NaN in
 * the reference partition's K or V (torch.min / max propagate it). Where an fp32 intermediate overflows, which only bf16
 * inputs can cause (a reference range hi - lo beyond the fp32 range, or one so small that x or its square overflows),
 * the scores depart from the definition, and an overflowing sigma makes the whole partition NaN.
 * The reference evaluates the chain in the cache dtype; here it is fp32, rounded once. Ties in the rank go to the earlier
 * position. 1 <= lag_size <= 1024 (kLagMax), every head_dim the problem validates. V must be device memory.
 * Check order (the first failure is returned): validate the problem -> n_kept == 0 returns KVP_OK (compress) ->
 * K / V / K_out / V_out null and alignment (compress) -> K, V, scores_out null and K / V alignment (score call) ->
 * n_sink < 0 or lag_size < 1 gives KVP_ERR_BAD_ARGUMENT -> lag_size > 1024 gives KVP_ERR_UNSUPPORTED_SHAPE ->
 * workspace. One kernel writes the scores and the selection keys; a compress takes 3 launches (memset, score,
 * select+compact) and keeps the n_kept best scores (scores_out nullable). Memory beyond the workspace: none. */
int kvp_lagkv_score(const kvp_problem* p, const void* K, const void* V, int32_t n_sink, int32_t lag_size,
                    int32_t cross_scoring, void* scores_out, void* workspace, size_t workspace_bytes,
                    kvp_stream_t stream);
int kvp_lagkv_compress(const kvp_problem* p, const void* K, const void* V, int32_t n_sink, int32_t lag_size,
                       int32_t cross_scoring, void* K_out, void* V_out, int32_t* idx_out, void* scores_out,
                       void* workspace, size_t workspace_bytes, kvp_stream_t stream);

/* ---- CURPress (kvpress/presses/cur_press.py, CurDKV, https://arxiv.org/abs/2509.15038) ------------------------------
 * Reads K and V only. Per row (b, kv head j) with S positions and w = local_window_size, evaluated in fp32 from the
 * 16-bit inputs and rounded once to the cache dtype:
 *   - a_k(s) = sum_d k_d^2, or with a projection G [D, r] (float32, row-major, device memory):
 *     a_k(s) = sum_c (sum_d k_d G_dc)^2. a_v(s) likewise from V. G == NULL and r == 0: no projection.
 *   - w >= 1: window c covers [cw, (c+1)w) within [0, S), and p_k(s) = a_k(s) / sum_{t in window} a_k(t) with IEEE
 *     rules (0/0 = NaN). The last, short window sums its real positions only (the reference pads with zeros).
 *     w == 0: no local approximation, p_k = a_k. p_v likewise.
 *   - u(s) = p_k, p_v, (p_k + p_v) / 2 or p_k p_v for leverage_type 0, 1, 2, 3 (the reference's "key", "value",
 *     "kv_avg", "kv_product"). Type 0 does not read V and type 1 does not read K.
 *   - T = sum_s u(s) over all S positions, the sinks included; score(s) = u(s) / T; then positions s < num_sinks score
 *     exactly 1 (num_sinks >= S: all of them; 0: none).
 * NaN and inf propagate as in torch: one NaN u makes T, and so every non-sink score of the row, NaN. A window whose a_k
 * (or a_v) is all zero is 0/0 = NaN, as in the reference; a zero row inside a non-zero window scores 0. An inf u makes T
 * inf, its own score NaN and the other scores 0. The evaluation is fp32: where a sum of squares, or the product of two
 * of them without local approximation, leaves the fp32 range, which only bf16 inputs near the top of their range can
 * cause, the scores depart from the definition. The shared selection ranks a NaN score above every number, the sinks' 1
 * included, and breaks ties by position: a NaN row keeps its first non-sink positions, and its sinks only once every
 * other position is kept. The windows are relative to the first row of the K / V view, so a slice of a cache gets its
 * own windows. The reference evaluates the chain in the cache dtype
 * and raises on 16-bit caches with a projection (a 16-bit matrix times a float32 one); here the projection is fp32.
 * 0 <= local_window_size <= 1024, 0 <= r <= 32, every head_dim the problem validates. G needs only float alignment.
 * Check order (the first failure is returned): validate the problem -> n_kept == 0 returns KVP_OK (compress) ->
 * K / V / K_out / V_out null and alignment (compress) -> K, V, scores_out null and K / V alignment (score call) ->
 * num_sinks < 0, leverage_type outside 0..3, local_window_size < 0, r < 0 or (G == NULL) != (r == 0) give
 * KVP_ERR_BAD_ARGUMENT -> local_window_size > 1024 or r > 32 gives KVP_ERR_UNSUPPORTED_SHAPE -> workspace.
 * The workspace holds u as fp32 [B, Hkv, S] and one fp64 partial sum per 256 or more positions, summed in a fixed
 * order, so scores are bitwise independent of the schedule and of the batch. A compress takes 4 launches (memset, unit
 * sums, finalize, select+compact) and keeps the n_kept best scores (scores_out nullable). Memory beyond the workspace:
 * none. */
int kvp_cur_score(const kvp_problem* p, const void* K, const void* V, int32_t num_sinks, int32_t leverage_type,
                  int32_t local_window_size, const float* G, int32_t r, void* scores_out, void* workspace,
                  size_t workspace_bytes, kvp_stream_t stream);
int kvp_cur_compress(const kvp_problem* p, const void* K, const void* V, int32_t num_sinks, int32_t leverage_type,
                     int32_t local_window_size, const float* G, int32_t r, void* K_out, void* V_out, int32_t* idx_out,
                     void* scores_out, void* workspace, size_t workspace_bytes, kvp_stream_t stream);

/* ---- MergingPress (kvpress/presses/merging_press.py) ----------------------------------------------------------------
 * Keeps the same rows as hard eviction, but first folds every evicted value into the kept row whose key is most
 * cosine-similar. Keys are only gathered, so the press is safe under RoPE. Per row (b, kv head j):
 *   - kept: the n_kept kept positions, ascending and distinct, numbered by kept slot t; ev: the other n_evict = S - n_kept
 *     positions, ascending, numbered by evicted slot e.
 *   - sim(e, t) = (K[e].K[t]) / (max(|K[e]|, 1e-6) max(|K[t]|, 1e-6)), from the raw 16-bit keys: exact products, fp32
 *     accumulation, fp32 norms.
 *   - target(e) is the kept slot with the largest sim; exact ties go to the lowest slot (the lowest position). A NaN
 *     similarity wins the max, as in torch.max: the first NaN column is the target. max_sim(e) = sim(e, target(e)).
 *   - The gate: ok(e) = max_sim(e) >= similarity_threshold. If merge_fraction < 1: thr = torch.quantile over the row's
 *     n_evict entries of max_sim with the non-ok entries at -inf, at q = 1 - merge_fraction, and ok &= max_sim >= thr.
 *     torch's arithmetic is reproduced exactly: q rounded to fp32, rank = q (n_evict - 1) in fp32, the order statistics
 *     at trunc(rank) and ceil(rank), and torch.lerp's two-branch formula (weight below 0.5: below + w (above - below),
 *     else above - (above - below)(1 - w), each one fused multiply-add). Two -inf order statistics give thr = NaN, and
 *     no entry of that row merges (q = 0.25 over [-inf, -inf, 0.2, 0.5, 0.9]).
 *   - w(e) = clamp(max_sim, min=0) ok |V[e]| / (|V[e]| + |V[target]| + 1e-6), in this order in fp32 (|V| in fp32).
 *   - acc_v(t) = sum of w(e) V[e] and acc_w(t) = sum of w(e) over the e with target(e) = t, both fp32, each product
 *     rounded, in ASCENDING e (the order of the reference's CPU scatter_add_). Where acc_w > 0:
 *     V_out[t] = (V[t] + acc_v) / (1 + acc_w), rounded once to the cache dtype; everywhere else V[t] bit for bit.
 * NaN / inf: a NaN or inf key makes its similarities NaN (inf / inf), so a NaN or inf evicted key targets slot 0 and a
 * NaN or inf kept key is the target of every evicted row whose earlier columns are numbers. A NaN max_sim never passes
 * the gate but gives a NaN weight (clamp keeps NaN, NaN * 0 = NaN): its target's acc_w is NaN, and that row is left
 * unmerged. So does an inf or NaN evicted value, whose norm makes its weight NaN, as in the reference.
 * A zero key has similarity 0 with every column, so it targets slot 0 and passes a threshold of 0.
 * Outputs: target_out (int32) and sim_out (fp32), both nullable, [B, Hkv, n_evict] contiguous: target and max_sim by
 * evicted slot, target in kept-slot numbering. Two calls give bitwise-equal outputs, and a row's outputs do not depend
 * on the batch it is in.
 * kvp_merging_compress: the selection of kvp_scores_compress on `scores` (K_out, V_out, idx_out as there), then the merge
 *   rewrites the n_kept rows of V_out. kvp_workspace_bytes(KVP_SCORER_MERGING) sizes its workspace; a compress takes 7
 *   launches (memset, keys, select+compact, prologue, argmax, plan, merge), 6 when nothing is evicted.
 * kvp_merging_merge: kept_idx int32 [B, Hkv, n_kept] contiguous, ascending and distinct in [0, S) (not checked);
 *   V_out contiguous [B, Hkv, n_kept, D] gets the merged kept rows. Same workspace; 4 launches; K_out is not written.
 * similarity_threshold in [0, 1] and merge_fraction in (0, 1], else KVP_ERR_BAD_ARGUMENT (NaN included). Every head_dim
 * the problem validates. Memory beyond the workspace: none; no n_evict x n_kept tensor is formed.
 * Check order (the first failure is returned): validate the problem -> (compress) n_kept == 0 returns KVP_OK ->
 * K / V / K_out / V_out null and 16-byte alignment (compress) -> scores / score_stride null (compress); K, V, kept_idx,
 * V_out null (merge) -> K, V, V_out 16-byte and kept_idx 4-byte alignment (merge) -> target_out, sim_out 4-byte alignment
 * -> similarity_threshold -> merge_fraction -> workspace. A merge call with n_kept == 0 enqueues nothing. */
int kvp_merging_compress(const kvp_problem* p, const void* scores, const int64_t* score_stride, const void* K,
                         const void* V, float similarity_threshold, double merge_fraction, void* K_out, void* V_out,
                         int32_t* idx_out, int32_t* target_out, float* sim_out, void* workspace,
                         size_t workspace_bytes, kvp_stream_t stream);
int kvp_merging_merge(const kvp_problem* p, const void* K, const void* V, const int32_t* kept_idx,
                      float similarity_threshold, double merge_fraction, void* V_out, int32_t* target_out,
                      float* sim_out, void* workspace, size_t workspace_bytes, kvp_stream_t stream);

/* ---- ThinKPress (kvpress/presses/think_press.py, https://arxiv.org/abs/2407.21018) -----------------------------------
 * Zeroes the key CHANNELS that matter least to the last window queries, in place; no position is removed. Per row
 * (b, kv head j), with G = Hq / Hkv, w = window and S positions:
 *   qn(c)    = 1/(G w) sum_{g<G} sum_{i<w} q_window[b, jG+g, i, c]^2    (the query heads jG ... jG+G-1 of kv head j)
 *   kn(c)    = 1/S sum_{s<S} K[b, j, s, c]^2
 *   score(c) = qn(c) kn(c), an fp32 value
 * The D - n_pruned largest scores are kept: at equal scores the lower channel is kept, and NaN ranks above every number
 * (torch.topk), NaNs among themselves by channel. Every element of a pruned channel, at every position of the view, is
 * set to +0.0 (bit pattern 0); every other element of K is left bit for bit. V is neither read nor written.
 * Evaluation order: the squares of the 16-bit inputs are exact. kn: per block of 256 positions (fixed by S alone) fp32
 * sums, each element passing through at most 68 fp32 additions; the blocks summed in ascending order in fp64, then / S.
 * qn: fp64 sums in a fixed order, / (G w). score = (qn kn) evaluated in fp64, rounded once to fp32. Against the same
 * definition in float64 (fp32 rounding of the exact product included), for S < 2^31 and G w < 2^31:
 *   |score - score64| <= 2^-16 |score64|  (+ 2^-149 per position for bf16 keys below 2^-63 in magnitude)
 * NaN / inf: a NaN key or query element makes its channel's score NaN; an inf key (or query) makes it inf, or NaN when
 * the other factor is 0 (inf * 0). Only bf16 keys can leave the fp32 range: an element of magnitude 2^64 or more, or a
 * channel's 256-position block sum beyond 3.4e38, makes kn inf where the float64 definition is finite; a product qn kn
 * beyond the fp32 range is inf in the definition too. The scores, the pruned set and the zeroed K of a row are bitwise
 * independent of the SM count, of the batch the row sits in and of the strides.
 * Arguments:
 *   K          [B, Hkv, S, D] in place, through p->k_stride; any strided view the problem validates. Nothing outside
 *              the view is written. p->v_stride is ignored (K's strides are validated in its place); p->n_kept is
 *              unused (callers pass S) but validated as usual.
 *   q_window   RoPE'd queries [B, Hq, window, D], contiguous, in K's dtype, 16-byte aligned.
 *   pruned_out nullable, int32 [B, Hkv, n_pruned], the pruned channels ascending.
 *   channel_scores_out nullable, float32 [B, Hkv, D], the scores.
 * Every head_dim the problem validates, every G and window >= 1.
 * Check order (the first failure is returned): p null -> validate the problem -> window >= 1 and 0 <= n_pruned <= D, else
 * KVP_ERR_BAD_ARGUMENT -> n_pruned == 0 returns KVP_OK and enqueues nothing (the outputs are not written) -> K, q_window
 * null -> K, q_window 16-byte and pruned_out, channel_scores_out 4-byte alignment -> workspace null -> its 16-byte
 * alignment -> its size. kvp_workspace_bytes(KVP_SCORER_THINK) is 4 R + 32 R + 4 R ceil(S / 256) D bytes, each region
 * rounded up to 256 (R = B Hkv): row tickets, the pruned-channel bitmask and the per-block partial sums. A call takes 3
 * launches (memset of the tickets, reduce + select, zero). Memory beyond the workspace: none.
 * The return type is kvp_status, an int-sized enum with the values of every other entry point's int. */
kvp_status kvp_think_prune(const kvp_problem* p, void* K, const void* q_window, int32_t window, int32_t n_pruned,
                           int32_t* pruned_out, float* channel_scores_out, void* workspace, size_t workspace_bytes,
                           kvp_stream_t stream);

/* ---- FinchPress (kvpress/presses/finch_press.py, https://direct.mit.edu/tacl/article/doi/10.1162/tacl_a_00716) ------
 * SnapKV with the window set by the prompt: the w queries after the user's delimiter (the question) score the context
 * and are always kept. Per row (b, kv head j), with G = Hq / Hkv and the window queries at positions S - w + i:
 *   P[h, i, s]  = softmax over all S keys of q_window[b, h, i] . K[b, j, s] / sqrt(D), causal inside the window
 *   c_i         = S - w + i if normalize != 0, else 1
 *   score(s)    = 1/(G w) sum_{g<G} sum_{i<w} c_i P[b, jG+g, i, s]     for the context positions s < S - w
 * evaluated in fp32 and rounded once to the cache dtype (a score beyond the fp16 range is +inf, as in the reference).
 * The scale is 1/sqrt(D), as in the reference's compute_window_attention. Deviation: c_i is the exact integer; the
 * reference multiplies its cache-dtype weights by an int64 arange, which rounds c_i to the cache dtype (8 significant
 * bits in bf16; inf from 65520 on in fp16, which makes its scores inf or NaN). scores_out (nullable) holds the scores
 * and, at the w window positions, the reference's sentinel: the largest context score of the whole call + 1, rounded
 * to the cache dtype. The selection forces the window instead (as SnapKV's), so it is kept even where max + 1 rounds
 * back to max.
 * Selection of kvp_finch_compress:
 *   - chunk_length == 0: the n_kept best positions of the row (chunk_kept and tail_kept are ignored).
 *   - chunk_length > 0: chunk c covers [c L, min(S, (c+1) L)), L = chunk_length. Each of the n_full = S / L full chunks
 *     keeps its chunk_kept best positions, the short last chunk (S mod L positions, if any) its tail_kept best; a window
 *     position in the short last chunk competes for that chunk's budget. The host computes the counts (the reference's
 *     max(1, int(len (1 - r)))); n_kept must be n_full chunk_kept + tail_kept.
 *   Ties go to the lowest positions; the kept rows come out in ascending position order.
 *   - inv_freq (nullable, fp32 [D/2]): the key kept at position s that lands in output row j is re-rotated by
 *     (j - s) inv_freq with kvp_scores_compress_rerotate's rounding points; values are copied exactly. With a null
 *     inv_freq K_out and V_out are exact gathers.
 * q_window: RoPE'd window queries [B, Hq, w, D], contiguous, in K's dtype, 16-byte aligned; 1 <= w < S.
 * Instantiated for bf16 / fp16, D in {64, 128} and 1 <= G <= 8; other shapes give KVP_ERR_UNSUPPORTED_SHAPE (FinchPress
 * scores them with blocked cuBLAS GEMMs and selects through kvp_scores_compress_chunked). Indexing is 64-bit. Every sum
 * has a fixed order that depends on (S, w, G, D) only: two calls give bitwise-equal results, and a row's scores do not
 * depend on the batch or the strides.
 * Check order (the first failure is returned): validate the problem -> (compress) n_kept == 0 returns KVP_OK ->
 * (compress) K / V / K_out / V_out null and 16-byte alignment -> K (score), q_window, scores_out (score) null ->
 * K (score), q_window 16-byte alignment -> w < 1 or w >= S gives KVP_ERR_BAD_ARGUMENT -> (compress) chunk_length < 0,
 * or with chunk_length > 0: chunk_kept outside [1, L] while n_full > 0, tail_kept outside [1, S mod L] (0 when L
 * divides S) or n_kept != n_full chunk_kept + tail_kept gives KVP_ERR_BAD_ARGUMENT -> D not 64 / 128 or G > 8 gives
 * KVP_ERR_UNSUPPORTED_SHAPE -> workspace null -> its 16-byte alignment -> its size.
 * kvp_workspace_bytes(KVP_SCORER_FINCH) sizes the largest window, w = S - 1: the selection regions every scorer has,
 * plus 4 R S (chunked selection: kept positions) + 8 B Hq (64 qpos + w) (softmax partials; qpos = 128 for G = 1, else
 * 64) + 4 B Hq w (normalisers) + 4 R S_pad (column sums), each region rounded up to 256 bytes (R = B Hkv, S_pad = S
 * rounded up to 256). A compress takes 6 launches unchunked (memset, stats, merge, column sums, finalize,
 * select+compact) and 7 chunked (the selection is a chunk select and a gather); scores_out adds the sentinel fill.
 * Memory beyond the workspace: none; no [Hq, w, S] tensor is formed.
 * The return type is kvp_status, an int-sized enum with the values of every other entry point's int. */
kvp_status kvp_finch_score(const kvp_problem* p, const void* K, const void* q_window, int32_t window, int32_t normalize,
                           void* scores_out, void* workspace, size_t workspace_bytes, kvp_stream_t stream);
kvp_status kvp_finch_compress(const kvp_problem* p, const void* K, const void* V, const void* q_window, int32_t window,
                              int32_t normalize, int32_t chunk_length, int32_t chunk_kept, int32_t tail_kept,
                              const float* inv_freq, void* K_out, void* V_out, int32_t* idx_out, void* scores_out,
                              void* workspace, size_t workspace_bytes, kvp_stream_t stream);
/* The chunked selection of kvp_finch_compress on caller scores [B, Hkv, S] (K's dtype, element strides score_stride for
 * (b, h), s contiguous), with inv_freq nullable as there (D a multiple of 16 when given). Check order: validate the
 * problem -> n_kept == 0 returns KVP_OK -> K / V / K_out / V_out null and alignment -> scores, score_stride null ->
 * chunk_length < 1 or the chunk counts as above give KVP_ERR_BAD_ARGUMENT -> inv_freq with D not a multiple of 16
 * gives KVP_ERR_UNSUPPORTED_SHAPE -> workspace (kvp_workspace_bytes(KVP_SCORER_FINCH) is enough). 4 launches (memset,
 * keys, chunk select, gather). */
kvp_status kvp_scores_compress_chunked(const kvp_problem* p, const void* scores, const int64_t* score_stride,
                                       int32_t chunk_length, int32_t chunk_kept, int32_t tail_kept, const void* K,
                                       const void* V, const float* inv_freq, void* K_out, void* V_out,
                                       int32_t* idx_out, void* workspace, size_t workspace_bytes,
                                       kvp_stream_t stream);

/* ---- CAMPress (kvpress/presses/cam_press.py, CaM, https://openreview.net/forum?id=LCTmppB165) ----------------------
 * DecodingPress's compaction with merge-before-prune: some evicted values are folded into the kept rows that follow
 * them, with a probability set by the running sum of the attention each position received while decoding. One
 * compaction of one layer, per batch element b (all kv heads share one selection, as in the reference), with the
 * base press's scores [B, Hkv, S] (cache dtype), the fp32 running sum A [B, Hkv, S], n_kept = target_size,
 * n_merge = min(k, S - n_kept) (k: the layer's steps since its last compaction), merge_budget >= 1 and caller uniforms
 * u [B, Hkv, n_merge] in [0, 1):
 *   1. m[s] = (sum of the Hkv scores in ascending head order, fp32) / Hkv, rounded once to the cache dtype.
 *   2. kept: the n_kept largest m, ranked as kvp_scores_compress ranks 16-bit keys (NaN above every number, -0 == +0),
 *      ties to the LOWEST positions; kept[0 .. n_kept) ascending. evicted: exactly the other S - n_kept positions.
 *   3. candidates: the n_merge evicted positions ranked first by (m descending, position descending), NaN above every
 *      number (the reference's flip + stable argsort: ties go to the LATER position; under StreamingLLM every evicted
 *      m is 0 and the candidates are the n_merge evicted positions just before the recent window); e[0 .. n_merge)
 *      ascending.
 *   4. t_i = the number of kept positions below e_i; the window of candidate i is the kept ranks
 *      [t_i, min(t_i + merge_budget, n_kept)), n_i its size (0 when e_i is above every kept position).
 *   5. per head j: mean_i = (sum of A[kept[r]] over the window, ascending r, fp32) / max(n_i, 1);
 *      p_i = A[e_i] / mean_i with NaN -> 0 (0 / 0: a zero running sum) and +inf -> 1 (a zero mean under a positive
 *      A[e_i]), then clamped to [0, 1]; mask_i = u[b, j, i] < p_i, a Bernoulli(p_i) draw reproducible from u.
 *   6. for each kept rank r: K_out[r] = K[kept[r]] and attn_out[r] = A[kept[r]] exactly;
 *      V_out[r] = round(V[kept[r]] + sum of (mask_i / n_i) V[e_i] over the candidates whose window holds r, ascending i),
 *      accumulated in fp32 from V[kept[r]], each term one fused multiply-add, rounded once to the cache dtype.
 *   A row can receive far more than merge_budget terms: under StreamingLLM all n_merge candidates share one t_i, so
 *   each of the first merge_budget recent rows receives all of them. The kernels assume no bound but n_merge.
 * Deviations from the reference: the running sum is fp32, not the cache dtype; the evicted set is the complement of
 * the kept set (the reference's two topk calls can make a tied position both kept and evicted, or neither); the merge
 * sums are fp32, in a fixed order and rounded once, not a bf16 atomic scatter_add_; ties among the kept rows go to the
 * lowest positions. With fp32 inputs the reference computes in fp32, and steps 1-6 agree with it to fp32 rounding.
 * NaN / inf: a NaN score ranks above every number in both selections. A non-finite A gives p_i by the rules above. A
 * non-finite evicted value reaches every row of its window even when its draw fails (0 * inf = NaN), as in the
 * reference. Against the float64 definition (the same kept set, candidates and draws),
 *   |V_out[r] - V64[r]| <= ulp(V64[r]) / 2 + (c_r + 2) 2^-24 (|V[kept[r]]| + sum of (mask_i / n_i) |V[e_i]|)
 * elementwise, c_r being the number of terms of row r.
 * Arguments:
 *   scores      [B, Hkv, S] in K's dtype, element strides score_stride (b, h), s contiguous, 2-byte aligned.
 *   attn_sum    fp32 [B, Hkv, S], element strides attn_stride (b, h), s contiguous: the view may sit in a capacity
 *               buffer. attn_out likewise [B, Hkv, n_kept] with attn_out_stride; it must not overlap attn_sum.
 *   uniforms    fp32 [B, Hkv, n_merge] contiguous; may be null when n_merge == 0.
 *   K_out, V_out contiguous [B, Hkv, n_kept, D].
 *   idx_out     nullable, int32 [B, n_kept]: the kept positions, ascending.
 *   merge_idx_out nullable, int32 [B, n_merge]: the candidates e, ascending.
 *   merge_prob_out nullable, fp32 [B, Hkv, n_merge]: p_i.
 * Every head_dim the problem validates. Indexing is 64-bit. Every sum has a fixed order: two calls give bitwise-equal
 * results, and a row's results do not depend on the batch, the SM count or the strides.
 * Check order (the first failure is returned): validate the problem -> n_kept == 0 returns KVP_OK and enqueues nothing
 * -> K / V / K_out / V_out null and 16-byte alignment -> scores, score_stride, attn_sum, attn_stride, attn_out,
 * attn_out_stride null, uniforms null with n_merge != 0 -> scores 2-byte and attn_sum, attn_out, uniforms, idx_out,
 * merge_idx_out, merge_prob_out 4-byte alignment -> merge_budget < 1 or n_merge outside [0, S - n_kept] gives
 * KVP_ERR_BAD_ARGUMENT -> workspace null -> its 16-byte alignment -> its size.
 * kvp_workspace_bytes(KVP_SCORER_CAM) does not depend on n_merge or merge_budget: the selection regions of B rows
 * (kvp_scores_select's for a [B, 1, S] problem), then 4 B n_kept (kept positions) + 4 B (S - n_kept) twice
 * (candidates, t) + 4 B Hkv (S - n_kept) (weights mask_i / n_i), each region rounded up to 256 bytes. A call takes 6
 * launches (memset, head mean + keys, select, candidates, probabilities, merge + compaction), 4 when n_merge == 0.
 * Memory beyond the workspace: none.
 * The return type is kvp_status, an int-sized enum with the values of every other entry point's int. */
kvp_status kvp_cam_compress(const kvp_problem* p, const void* scores, const int64_t* score_stride, const void* K,
                            const void* V, const float* attn_sum, const int64_t* attn_stride, int32_t n_merge,
                            int32_t merge_budget, const float* uniforms, void* K_out, void* V_out, float* attn_out,
                            const int64_t* attn_out_stride, int32_t* idx_out, int32_t* merge_idx_out,
                            float* merge_prob_out, void* workspace, size_t workspace_bytes, kvp_stream_t stream);

/* ---- KVzapPress (kvpress/presses/kvzap_press.py, https://arxiv.org/abs/2601.07891) ---------------------------------
 * Scores from a small per-layer surrogate model of the attention module's input hidden states x [B, S, hidden] (S =
 * p->S); no queries, attention weights or K / V are read. Per (b, kv head j, s), with gelu(t) = t/2 (1 + erf(t/sqrt 2))
 * (nn.GELU's default) and every weight in the cache dtype p->dtype:
 *   hd > 0 (MLP):    score = b2[j] + sum_c W2[j, c] gelu(b1[c] + sum_k W1[c, k] x[b, s, k])
 *                    W1 [hd, hidden], b1 [hd], W2 [Hkv, hd], b2 [Hkv], contiguous as nn.Linear stores them.
 *   hd == 0 (linear): score = b[j] + sum_k W[j, k] x[b, s, k], with W [Hkv, hidden] passed as w1, b [Hkv] as b1;
 *                    w2 and b2 are not read.
 * Every sum is fp32 in an order fixed by the shape: the pre-activation is the K-ordered tensor-core accumulation
 * (B S > 32) or the CUDA-core sum of 8-element slices added lane by lane, then across the warp (B S <= 32); then
 * b1 and the GELU in fp32; the W2 products are added per chunk of 128 units (8 when B S <= 32), the chunks in
 * ascending order, then b2. The score is rounded ONCE to the cache dtype and written into scores_out
 * [B, Hkv, S] contiguous.
 * Deviation from the reference: it evaluates Linear -> GELU -> Linear in the cache dtype and rounds after each layer;
 * here nothing is rounded between the layers. Against the float64 evaluation s64 of the same 16-bit inputs, with
 * a_c = b1[c] + sum_k W1[c, k] x_k, A_c = |b1[c]| + sum_k |W1[c, k] x_k|, e_c = (hidden + 2) 2^-22 A_c,
 * E_c = 1.2 e_c + 2^-20 (|a_c| + e_c) and h_c = gelu(a_c),
 *   |score_fp32 - s64| <= E = sum_c |W2[j, c]| E_c + (hd + 260) 2^-23 (|b2[j]| + sum_c |W2[j, c]| (|h_c| + E_c))
 * (linear: E = (hidden + 2) 2^-22 (|b[j]| + sum_k |W[j, k] x_k|)), so the score lies in [RD(s64 - E), RU(s64 + E)],
 * RD / RU rounding down / up to the cache dtype. Two calls give bitwise-equal scores, and a row's score does not
 * depend on the other rows, the strides or the SM count (it does on whether B S <= 32, which picks the order above).
 * Arguments:
 *   x        [B, S, hidden] in the cache dtype, element strides x_stride (b, s), the hidden dim contiguous, 16-byte
 *            aligned; a stride of a size-1 dim is not read.
 *   w1       16-byte aligned; b1, w2, b2 2-byte aligned.
 * Supported: hidden a multiple of 8 up to 16384, hd 0 or a multiple of 8 up to 2048, Hkv up to 32, both dtypes;
 * anything else is KVP_ERR_UNSUPPORTED_SHAPE (the press then scores with cuBLAS in fp32).
 * Check order (the first failure is returned): validate the problem -> (compress) n_kept == 0 returns KVP_OK and
 * enqueues nothing -> (compress) K / V / K_out / V_out null and 16-byte alignment -> (score) scores_out null ->
 * scores_out 2-byte alignment -> x, x_stride, w1, b1 null, and w2, b2 null when hd > 0 -> x, w1 16-byte and b1, w2,
 * b2 2-byte alignment -> hidden < 1 or hd < 0 gives KVP_ERR_BAD_ARGUMENT -> x_stride negative or not a multiple of 8,
 * or x_stride[1] < hidden with S > 1, gives KVP_ERR_BAD_STRIDE -> the supported shapes -> workspace null -> its
 * 16-byte alignment -> its size.
 * kvp_workspace_bytes(KVP_SCORER_KVZAP): the selection regions (as kvp_scores_compress), then
 * 4 B P Hkv B S for the partials, P = 256 when B S <= 32 and 16 otherwise (enough for hd = 2048), then 2 B B Hkv S
 * for the scores a compress call selects on, each region rounded up to 256 bytes. kvp_launches_per_compress says 5
 * (memset, scores, reduce of the partials, keys, select + compact); the linear model takes 4 (no reduce), a score
 * call 2 (MLP) or 1 (linear). Memory beyond the workspace: none.
 * The return type is kvp_status, an int-sized enum with the values of every other entry point's int. */
kvp_status kvp_kvzap_score(const kvp_problem* p, const void* x, const int64_t* x_stride, int32_t hidden, int32_t hd,
                           const void* w1, const void* b1, const void* w2, const void* b2, void* scores_out,
                           void* workspace, size_t workspace_bytes, kvp_stream_t stream);
/* The scores above, then the selection and compaction of kvp_scores_compress: 16-bit keys, NaN above every number,
 * -0 == +0, ties to the lowest positions. scores_out is nullable here. */
kvp_status kvp_kvzap_compress(const kvp_problem* p, const void* x, const int64_t* x_stride, int32_t hidden, int32_t hd,
                              const void* w1, const void* b1, const void* w2, const void* b2, const void* K,
                              const void* V, void* K_out, void* V_out, int32_t* idx_out, void* scores_out,
                              void* workspace, size_t workspace_bytes, kvp_stream_t stream);

/* ---- DMSPress (kvpress/presses/dms_press.py): threshold eviction --------------------------------------------------
 * Every (b, h, s) with s < n_evict and scores[b, h, s] < threshold, for scores [B, Hkv, n] in dtype (bf16 / fp16),
 * element strides score_stride (b, h), s contiguous, 2-byte aligned. The comparison is made in the score dtype: the
 * threshold is first rounded to nearest-even in that dtype, as torch does for `scores < python_float` (a bf16 score
 * of 0.099609375 is not below 0.0998). NaN is never evicted; -0 is not below +0.
 * Output: b_out, h_out, s_out (int64, capacity B Hkv n_evict) get b, h and s + shift of every evicted position in
 * torch.where order (b, then h, then s ascending), and *count_out (int64, device) their number. The result is exact:
 * per-(row, 4096-position tile) counts, one scan, an ordered write, no atomics.
 * Check order: dtype -> B, Hkv, n < 1 or B Hkv ceil(n / 4096) >= 2^31 gives KVP_ERR_UNSUPPORTED_SHAPE -> n_evict outside [0, n]
 * gives KVP_ERR_BAD_ARGUMENT -> scores, score_stride, count_out null, and b_out, h_out, s_out null when n_evict > 0 ->
 * scores 2-byte alignment, negative strides, b_out, h_out, s_out, count_out 8-byte alignment (KVP_ERR_BAD_STRIDE) ->
 * workspace null -> its 16-byte alignment -> its size: 8 B Hkv ceil(n / 4096) bytes rounded up to 256 (the
 * per-tile counts).
 * 3 launches (counts, scan, write). Memory beyond the workspace: none.
 * The return type is kvp_status, an int-sized enum with the values of every other entry point's int. */
kvp_status kvp_threshold_evict(int32_t dtype, int32_t B, int32_t Hkv, int32_t n, const void* scores,
                               const int64_t* score_stride, int32_t n_evict, float threshold, int64_t shift,
                               int64_t* b_out, int64_t* h_out, int64_t* s_out, int64_t* count_out, void* workspace,
                               size_t workspace_bytes, kvp_stream_t stream);

/* ---- selection only: the n_kept best positions of every [S] score row, ascending, into idx_out
 * [B, Hkv, n_kept]; no K/V are touched (p->D and the K/V strides are ignored). What head-wise presses need:
 * AdaKVPress (kvpress/presses/adakv_press.py:53-78) = this call on the [B, Hkv, S] scores with n_safe, then
 * on the negated, head-flattened [B, 1, Hkv*S] scores with the number of positions to prune. */
int kvp_scores_select(const kvp_problem* p, const void* scores, const int64_t* score_stride,
                      int32_t* idx_out, void* workspace, size_t workspace_bytes, kvp_stream_t stream);

/* ---- KeyRerotationPress (SURVEY §8f, first "next" row): same selection as kvp_scores_compress, but each
 * kept key is re-rotated from its original position s to its new position j (kvpress/presses/
 * key_rerotation_press.py:50-152): k * cos((j-s) inv_freq) + rotate_half(k) * sin((j-s) inv_freq).
 * inv_freq: fp32 [D/2] (module.rotary_emb.inv_freq); D must be a multiple of 16. Values are copied as is. */
int kvp_scores_compress_rerotate(const kvp_problem* p, const void* scores, const int64_t* score_stride,
                                 const void* K, const void* V, const float* inv_freq, void* K_out,
                                 void* V_out, int32_t* idx_out, void* workspace,
                                 size_t workspace_bytes, kvp_stream_t stream);

/* Host buffers: every entry point takes DEVICE pointers (V may be pinned host memory for the scorers that do not read V to
 * score: the compaction kernel then gathers the kept V rows over PCIe). Staging whole caches from host memory through
 * these calls — per-kv-head chunks on three streams — is the host side's job: kvpress_b200/host_staging.py. */

#ifdef __cplusplus
}
#endif
#endif /* KVPRESS_B200_H */
