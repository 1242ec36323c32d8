// api.cu — the extern "C" surface declared in include/kvpress_b200.h.
// Validates the problem, carves the caller's workspace and enqueues the kernels on the caller's
// stream. Never allocates, never synchronises (except kvp_workspace_check), never throws.
#include <math.h>
#include <stdio.h>

#include <algorithm>
#include <atomic>
#include <cstddef>
#include <type_traits>

#include "common.cuh"

namespace kvp {

static thread_local char g_last_cuda_error[256] = "";

// kvp_status of a CUDA call. The KeyDiff, SnapKV, ExpectedAttention, CriticalKV, ObservedAttention, NonCausalAttention,
// LagKV, CUR and Finch score launchers report a shape they have no kernel for as cudaErrorNotSupported.
static int status(cudaError_t e, int scorer = KVP_SCORER_GENERIC) {
    if (e == cudaSuccess) return KVP_OK;
    if (e == cudaErrorNotSupported &&
        (scorer == KVP_SCORER_KEYDIFF || scorer == KVP_SCORER_SNAPKV || scorer == KVP_SCORER_EXPECTED_ATTENTION ||
         scorer == KVP_SCORER_CRITICALKV || scorer == KVP_SCORER_OBSERVED_ATTENTION ||
         scorer == KVP_SCORER_NON_CAUSAL_ATTENTION || scorer == KVP_SCORER_LAGKV || scorer == KVP_SCORER_CUR ||
         scorer == KVP_SCORER_FINCH))
        return KVP_ERR_UNSUPPORTED_SHAPE;
    snprintf(g_last_cuda_error, sizeof(g_last_cuda_error), "%s: %s", cudaGetErrorName(e), cudaGetErrorString(e));
    // launch-configuration errors are not sticky: clear them, or the cudaPeekAtLastError() of every later call
    // (of this library or of torch) would report this failure again
    cudaGetLastError();
    return KVP_ERR_CUDA;
}

static int validate(const kvp_problem* p, Dims* d, bool need_kv_strides = true) {
    if (p == nullptr) return KVP_ERR_NULL_POINTER;
    if (p->dtype != KVP_BF16 && p->dtype != KVP_F16) return KVP_ERR_UNSUPPORTED_DTYPE;
    if (p->B <= 0 || p->Hkv <= 0 || p->S <= 0 || p->D <= 0) return KVP_ERR_UNSUPPORTED_SHAPE;
    if (p->D % 8 != 0 || p->D > 256) return KVP_ERR_UNSUPPORTED_SHAPE;
    if (p->Hq <= 0 || p->Hq % p->Hkv != 0) return KVP_ERR_UNSUPPORTED_SHAPE;
    if (p->n_kept < 0 || p->n_kept > p->S) return KVP_ERR_BAD_ARGUMENT;
    if ((int64_t)p->B * p->Hkv > 65535) return KVP_ERR_UNSUPPORTED_SHAPE;  // gridDim.y
    if (need_kv_strides) {
        for (int i = 0; i < 3; ++i) {
            // rows must stay 16-byte aligned: every outer stride is a multiple of 8 elements
            if (p->k_stride[i] % 8 != 0 || p->v_stride[i] % 8 != 0) return KVP_ERR_BAD_STRIDE;
            if (p->k_stride[i] < 0 || p->v_stride[i] < 0) return KVP_ERR_BAD_STRIDE;
        }
        if (p->k_stride[2] < p->D || p->v_stride[2] < p->D) return KVP_ERR_BAD_STRIDE;
    }
    d->B = p->B;
    d->H = p->Hkv;
    d->Hq = p->Hq;
    d->S = p->S;
    d->D = p->D;
    d->n_kept = p->n_kept;
    d->R = p->B * p->Hkv;
    d->ks = {p->k_stride[0], p->k_stride[1], p->k_stride[2]};
    d->vs = {p->v_stride[0], p->v_stride[1], p->v_stride[2]};
    return KVP_OK;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// The window kvp_workspace_bytes / kvp_workspace_check size a scorer's scratch for: the largest a call may pass.
// ObservedAttention: n_q = S. Finch: w = S - 1 (at least 1). SnapKV: the most query rows G * window <= kSnapMaxRows
// with window < S (at least 1, so that a group too wide for any window still reaches the launcher's unsupported-shape
// status).
static int largest_window(const Dims& d, int scorer) {
    if (scorer == KVP_SCORER_OBSERVED_ATTENTION) return d.S;
    if (scorer == KVP_SCORER_FINCH) return std::max(1, d.S - 1);
    return std::max(1, std::min(kSnapMaxRows / (d.Hq / d.H), d.S - 1));
}

// The workspace of a call: sized when `base` is null, carved otherwise. `window` is SnapKV's or Finch's window, or the
// query rows n_q of ObservedAttention. Returns the total bytes and, in *zeroed, the
// leading bytes every call clears with one memset: the histograms, the counters and the tile prefixes. The
// histograms are whole KiB per row, so hist_lo and the counters follow hist_hi without padding.
static size_t layout(const Dims& d_call, int scorer, int window, void* base, Workspace* ws, size_t* zeroed) {
    const Dims d = scorer == KVP_SCORER_CAM ? cam_selection_dims(d_call) : d_call;
    Carve c(base);
    ws->R = d.R;
    if (scorer == KVP_SCORER_THINK) {  // no selection of positions: the channel statistics alone (think.cu)
        *ws = Workspace{};
        ws->R = d.R;
        ws->scorer_bytes = think_scratch_bytes(d);
        ws->scorer = c.take<char>(ws->scorer_bytes);
        *zeroed = 0;
        return c.bytes;
    }
    ws->n_tiles = (d.S + kTile - 1) / kTile;
    ws->S_pad = ws->n_tiles * kTile;
    ws->hist_hi = c.take<uint32_t>((size_t)d.R * 256);
    ws->hist_lo = c.take<uint32_t>((size_t)d.R * 256);
    ws->counters = c.take<uint32_t>((size_t)d.R * 3 + 64);
    ws->tile_prefix = c.take<uint2>((size_t)d.R * ws->n_tiles);
    *zeroed = c.bytes;
    ws->keys = c.take<uint16_t>((size_t)d.R * ws->S_pad);
    ws->tile_sfx = c.take<uint16_t>((size_t)d.R * ws->n_tiles * kSfxStride);
    ws->row_meta = c.take<uint2>(d.R);
    ws->scorer_bytes = scorer == KVP_SCORER_SNAPKV               ? snapkv_scratch_bytes(d, window)
                       : scorer == KVP_SCORER_EXPECTED_ATTENTION ? ea_scratch_bytes(d)
                       : scorer == KVP_SCORER_KEYDIFF            ? keydiff_scratch_bytes(d)
                       : scorer == KVP_SCORER_CRITICALKV         ? criticalkv_scratch_bytes(d)
                       : scorer == KVP_SCORER_OBSERVED_ATTENTION ? observed_attention_scratch_bytes(d, window)
                       : scorer == KVP_SCORER_NON_CAUSAL_ATTENTION ? non_causal_attention_scratch_bytes(d)
                       : scorer == KVP_SCORER_CUR                  ? cur_scratch_bytes(d)
                       : scorer == KVP_SCORER_MERGING              ? merging_scratch_bytes(d)
                       : scorer == KVP_SCORER_FINCH                ? finch_scratch_bytes(d, window)
                       : scorer == KVP_SCORER_CAM                  ? cam_scratch_bytes(d_call)
                       : scorer == KVP_SCORER_KVZAP                ? kvzap_scratch_bytes(d)
                                                                   : 0;
    ws->scorer = c.take<char>(ws->scorer_bytes);
    return c.bytes;
}

// One call on a carved workspace.
struct Call {
    Dims d;
    Workspace ws;
    size_t zeroed;  // see layout()
    cudaStream_t st;
    int carve(int scorer, int window, void* workspace, size_t bytes) {
        if (workspace == nullptr) return KVP_ERR_NULL_POINTER;
        if (!aligned16(workspace)) return KVP_ERR_BAD_STRIDE;
        return bytes < layout(d, scorer, window, workspace, &ws, &zeroed) ? KVP_ERR_WORKSPACE_TOO_SMALL : KVP_OK;
    }
    int zero() const { return status(cudaMemsetAsync(ws.hist_hi, 0, zeroed, st)); }
};

static int check_io(const void* K, const void* V, const void* K_out, const void* V_out) {
    if (!K || !V || !K_out || !V_out) return KVP_ERR_NULL_POINTER;
    if (!aligned16(K) || !aligned16(V) || !aligned16(K_out) || !aligned16(V_out))
        return KVP_ERR_BAD_STRIDE;
    return KVP_OK;
}

// K and V, where a compress call writes the kept rows, and how the selection stage treats them.
struct Io {
    const void* K;
    const void* V;
    void* K_out;
    void* V_out;
    int32_t* idx_out;
    const float* inv_freq;  // kvp_scores_compress_rerotate: the kept keys are re-rotated
    // where the selection writes the kept positions when idx_out is null and a later stage reads them (MergingPress)
    int32_t* (*kept_scratch)(const Dims&, const Workspace&) = nullptr;
    // chunk_length > 0: the chunked selection of FinchPress (kvp_finch_compress, kvp_scores_compress_chunked)
    int32_t chunk_length = 0, chunk_kept = 0, tail_kept = 0;
};

enum class Kind {
    compress,  // selects and compacts K / V
    select,    // kvp_scores_select: selects into idx_out; no K / V, so no K / V strides
    score,     // scores only: no n_kept == 0 short cut, no selection
};

// The checks of every call that carves a workspace, in the order they are made (the first failure is returned):
// validate -> n_kept == 0 short cut (compress, select) -> check_io (compress) -> the entry point's operand checks ->
// carve. A compress or select call with c->d.n_kept == 0 on return has nothing to do.
template <typename Operands>
static int prepare(Kind kind, const kvp_problem* p, int scorer, int window, const Io& io, Operands operands,
                   void* workspace, size_t workspace_bytes, kvp_stream_t stream, Call* c) {
    int rc = validate(p, &c->d, kind != Kind::select);
    if (rc) return rc;
    if (kind != Kind::score && c->d.n_kept == 0) return KVP_OK;
    if (kind == Kind::compress && (rc = check_io(io.K, io.V, io.K_out, io.V_out))) return rc;
    if ((rc = operands(c->d))) return rc;
    c->st = static_cast<cudaStream_t>(stream);
    return c->carve(scorer, window, workspace, workspace_bytes);
}

// prepare -> memset (unless zero == false) -> score -> selection (compress, select) -> after (compress).
// `score(const Call&)` enqueues the score stage and returns its cudaError_t; `after(const Call&, const int32_t* kept)`
// enqueues a stage on the selection's output (the kept positions) and returns its cudaError_t.
template <typename Operands, typename Score, typename After = std::nullptr_t>
static int run(Kind kind, const kvp_problem* p, int scorer, int window, const Io& io, Operands operands, Score score,
               void* workspace, size_t workspace_bytes, kvp_stream_t stream, bool zero = true, After after = nullptr) {
    Call c;
    int rc = prepare(kind, p, scorer, window, io, operands, workspace, workspace_bytes, stream, &c);
    if (rc || (kind != Kind::score && c.d.n_kept == 0)) return rc;
    if (zero && (rc = c.zero())) return rc;
    if ((rc = status(score(c), scorer))) return rc;
    if (kind == Kind::score) return KVP_OK;
    if (io.chunk_length > 0)
        return status(launch_select_compact_chunked(c.d, p->dtype, io.K, io.V, io.K_out, io.V_out, io.idx_out, c.ws,
                                                    io.chunk_length, io.chunk_kept, io.tail_kept,
                                                    finch_scratch_kept(c.d, c.ws), io.inv_freq, c.st));
    if (io.inv_freq)
        return status(launch_select_compact_rerotate(c.d, p->dtype, io.K, io.V, io.K_out, io.V_out, io.idx_out, c.ws,
                                                     io.inv_freq, c.st));
    int32_t* idx = io.idx_out != nullptr || io.kept_scratch == nullptr ? io.idx_out : io.kept_scratch(c.d, c.ws);
    if (kind == Kind::select) c.d.ks = c.d.vs = {0, 0, 0};
    if ((rc = status(launch_select_compact(c.d, io.K, io.V, io.K_out, io.V_out, idx, c.ws, c.st)))) return rc;
    if constexpr (!std::is_same<After, std::nullptr_t>::value) return status(after(c, idx), scorer);
    return KVP_OK;
}

static int no_operands(const Dims&) { return KVP_OK; }

enum class KnormPath { cluster, fused, two_kernels };

// The first KnormPath knorm_path may take; only kvp_debug_knorm_first_path changes it, so that the tests can run one
// input through every path.
static std::atomic<int> g_knorm_first_path{0};

// The kernels kvp_knorm_compress runs. `d` is null for a problem that failed validation: kvp_launches_per_compress
// still counts one, by its size alone.
static KnormPath knorm_path(const kvp_problem& p, const Dims* d) {
    const int first = g_knorm_first_path.load(std::memory_order_relaxed);
    // DecodingPress-sized caches: one launch of the cluster kernel (knorm_cluster.cu), no memset, no scratch
    if (first <= 0 && d != nullptr && knorm_cluster_applicable(*d)) return KnormPath::cluster;
    // Small caches beyond the cluster path are launch-latency-bound: one persistent kernel does score + select +
    // compact. Large caches measured faster as two kernels (the fused kernel's mixed read/write item stream costs
    // more HBM efficiency than the saved launch; K re-reads miss L2 anyway).
    constexpr size_t kFusedMaxBytes = (size_t)32 << 20;
    const size_t k_bytes = (size_t)p.B * p.Hkv * p.S * p.D * 2;
    return first <= 1 && k_bytes <= kFusedMaxBytes ? KnormPath::fused : KnormPath::two_kernels;
}

// The chunk counts of a chunked selection (chunk_length > 0), see kvp_finch_compress in the header.
static int chunk_counts_ok(const Dims& d, int32_t chunk_length, int32_t chunk_kept, int32_t tail_kept) {
    const int n_full = d.S / chunk_length, tail = d.S % chunk_length;
    if (n_full > 0 && (chunk_kept < 1 || chunk_kept > chunk_length)) return KVP_ERR_BAD_ARGUMENT;
    if (tail > 0 ? (tail_kept < 1 || tail_kept > tail) : tail_kept != 0) return KVP_ERR_BAD_ARGUMENT;
    const int64_t total = (int64_t)n_full * (n_full > 0 ? chunk_kept : 0) + tail_kept;
    return total == d.n_kept ? KVP_OK : KVP_ERR_BAD_ARGUMENT;
}

// Finch's window and instantiation checks, after its null / alignment checks and (compress) its chunk checks.
static int finch_window_ok(const Dims& d, int32_t window) {
    return window >= 1 && window < d.S ? KVP_OK : KVP_ERR_BAD_ARGUMENT;
}
static int finch_shape_ok(const Dims& d) {
    const int G = d.Hq / d.H;
    return (d.D == 64 || d.D == 128) && G <= 8 ? KVP_OK : KVP_ERR_UNSUPPORTED_SHAPE;
}

}  // namespace kvp

using namespace kvp;

extern "C" {

int kvp_abi_version(void) { return KVP_ABI_VERSION; }

const char* kvp_status_string(int status) {
    switch (status) {
        case KVP_OK: return "ok";
        case KVP_ERR_NULL_POINTER: return "null pointer";
        case KVP_ERR_UNSUPPORTED_SHAPE: return "unsupported shape";
        case KVP_ERR_UNSUPPORTED_DTYPE: return "unsupported dtype (bf16 / fp16 only)";
        case KVP_ERR_BAD_STRIDE: return "bad stride or alignment (rows must be 16-byte aligned)";
        case KVP_ERR_WORKSPACE_TOO_SMALL: return "workspace too small";
        case KVP_ERR_CUDA: return "CUDA error (see kvp_last_cuda_error)";
        case KVP_ERR_BAD_ARGUMENT: return "bad argument";
        case KVP_ERR_KERNEL_TIMEOUT: return "a kernel abandoned a bounded wait (outputs invalid)";
        default: return "unknown status";
    }
}

const char* kvp_last_cuda_error(void) { return g_last_cuda_error; }

int kvp_workspace_bytes(const kvp_problem* p, int scorer, size_t* bytes_out) {
    Dims d;
    int rc = validate(p, &d, false);
    if (rc) return rc;
    if (!bytes_out) return KVP_ERR_NULL_POINTER;
    // window only changes the SnapKV and ObservedAttention scratch; size for the largest supported window
    Workspace ws;
    size_t zeroed;
    *bytes_out = layout(d, scorer, largest_window(d, scorer), nullptr, &ws, &zeroed);
    return KVP_OK;
}

int kvp_workspace_check(const kvp_problem* p, int scorer, const void* workspace, size_t workspace_bytes,
                        kvp_stream_t stream) {
    Call c;
    int rc = validate(p, &c.d, false);
    if (rc || (rc = c.carve(scorer, largest_window(c.d, scorer), const_cast<void*>(workspace), workspace_bytes)))
        return rc;
    if (scorer == KVP_SCORER_THINK) return KVP_OK;  // its kernels have no bounded waits
    uint32_t flag = 0;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t e = cudaMemcpyAsync(&flag, c.ws.counters + kCounterErrSlot(c.ws.R), sizeof(flag),
                                    cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return status(e);
    return flag ? KVP_ERR_KERNEL_TIMEOUT : KVP_OK;
}

int kvp_launches_per_compress(const kvp_problem* p, int scorer, int* launches_out) {
    if (!p || !launches_out) return KVP_ERR_NULL_POINTER;
    switch (scorer) {
        case KVP_SCORER_STREAMING: *launches_out = 1; break;
        case KVP_SCORER_GENERIC: *launches_out = 3; break;  // memset, keys, select+compact
        case KVP_SCORER_KNORM: {  // cluster kernel | memset + (fused | score, select+compact)
            Dims d;
            const KnormPath path = knorm_path(*p, validate(p, &d, false) == KVP_OK ? &d : nullptr);
            *launches_out = path == KnormPath::cluster ? 1 : path == KnormPath::fused ? 2 : 3;
            break;
        }
        case KVP_SCORER_KEYDIFF: *launches_out = 5; break;  // memset, anchor partials, merge, score, select+compact
        case KVP_SCORER_SNAPKV: *launches_out = 5; break;  // memset, stats, colsum, finalize, select+compact
        // press defaults (use_covariance + use_vnorm): memset, logits (which also writes the value norms), finalize,
        // select+compact
        case KVP_SCORER_EXPECTED_ATTENTION: *launches_out = 4; break;
        // press defaults (first_stage_ratio > 0): memset, keys of the base scores, select n_first, score, force
        // n_first, memset, keys of the final scores, select+compact
        case KVP_SCORER_CRITICALKV: *launches_out = 8; break;
        case KVP_SCORER_OBSERVED_ATTENTION: *launches_out = 5; break;  // memset, stats, colsum, finalize, select+compact
        // memset, column sums, pooled partials, mean / std, z, select+compact
        case KVP_SCORER_NON_CAUSAL_ATTENTION: *launches_out = 6; break;
        case KVP_SCORER_LAGKV: *launches_out = 3; break;  // memset, scores + keys, select+compact
        case KVP_SCORER_CUR: *launches_out = 4; break;  // memset, unit sums, finalize, select+compact
        // memset, keys, select+compact, prologue, argmax (none when nothing is evicted), plan, merge
        case KVP_SCORER_MERGING: {
            Dims d;
            *launches_out = validate(p, &d, false) == KVP_OK && p->n_kept == p->S ? 6 : 7;
            break;
        }
        case KVP_SCORER_THINK: *launches_out = 3; break;  // memset, reduce + select, zero
        // unchunked: memset, stats, merge, column sums, finalize, select+compact (chunked: one more, see the header)
        case KVP_SCORER_FINCH: *launches_out = 6; break;
        // memset, head mean + keys, select, candidates, probabilities, merge + compaction (4 when n_merge == 0)
        case KVP_SCORER_CAM: *launches_out = 6; break;
        // memset, scores (gemm or W1-spread), reduce, keys, select+compact (the linear model: 4, no reduce)
        case KVP_SCORER_KVZAP: *launches_out = 5; break;
        default: return KVP_ERR_BAD_ARGUMENT;
    }
    return KVP_OK;
}

// ---- Knorm ---------------------------------------------------------------------------------------
int kvp_knorm_score(const kvp_problem* p, const void* K, void* scores_out, kvp_stream_t stream) {
    Dims d;
    int rc = validate(p, &d);
    if (rc) return rc;
    if (!K || !scores_out) return KVP_ERR_NULL_POINTER;
    if (!aligned16(K)) return KVP_ERR_BAD_STRIDE;
    Workspace ws = {};
    return status(launch_knorm_score(d, p->dtype, K, ws, scores_out, false, static_cast<cudaStream_t>(stream)));
}

int kvp_knorm_compress(const kvp_problem* p, const void* K, const void* V, void* K_out,
                       void* V_out, int32_t* idx_out, void* scores_out, void* workspace,
                       size_t workspace_bytes, kvp_stream_t stream) {
    const Io io = {K, V, K_out, V_out, idx_out, nullptr};
    Call c;
    int rc = prepare(Kind::compress, p, KVP_SCORER_KNORM, 0, io, no_operands, workspace, workspace_bytes, stream, &c);
    if (rc || c.d.n_kept == 0) return rc;
    const KnormPath path = knorm_path(*p, &c.d);
    if (path == KnormPath::cluster)
        return status(launch_knorm_cluster(c.d, p->dtype, K, V, K_out, V_out, idx_out, scores_out, c.st));
    if ((rc = c.zero())) return rc;
    if (path == KnormPath::fused) {
        // cudaErrorNotSupported: more work items than the fused kernel's queue addresses; two kernels instead
        const cudaError_t e = launch_knorm_fused(c.d, p->dtype, K, V, K_out, V_out, idx_out, scores_out, c.ws, c.st);
        if (e != cudaErrorNotSupported) return status(e);
    }
    if ((rc = status(launch_knorm_score(c.d, p->dtype, K, c.ws, scores_out, true, c.st)))) return rc;
    return status(launch_select_compact(c.d, K, V, K_out, V_out, idx_out, c.ws, c.st));
}

// Test hook, not in the public header: the first path knorm_path may take (0 = cluster, the default; 1 = fused;
// 2 = two kernels). Returns the previous value, or -1 (nothing changed) for any other `first`.
int kvp_debug_knorm_first_path(int first) {
    if (first < 0 || first > 2) return -1;
    return g_knorm_first_path.exchange(first, std::memory_order_relaxed);
}

// ---- KeyDiff -------------------------------------------------------------------------------------
int kvp_keydiff_score(const kvp_problem* p, const void* K, void* scores_out, void* workspace,
                      size_t workspace_bytes, kvp_stream_t stream) {
    auto operands = [&](const Dims&) {
        if (!K || !scores_out) return KVP_ERR_NULL_POINTER;
        return aligned16(K) ? KVP_OK : KVP_ERR_BAD_STRIDE;
    };
    auto score = [&](const Call& c) { return launch_keydiff_score(c.d, p->dtype, K, c.ws, scores_out, false, c.st); };
    // the score kernel writes no keys and no histogram when the selection is skipped: nothing to clear
    return run(Kind::score, p, KVP_SCORER_KEYDIFF, 0, {}, operands, score, workspace, workspace_bytes, stream, false);
}

int kvp_keydiff_compress(const kvp_problem* p, const void* K, const void* V, void* K_out, void* V_out,
                         int32_t* idx_out, void* scores_out, void* workspace, size_t workspace_bytes,
                         kvp_stream_t stream) {
    auto score = [&](const Call& c) { return launch_keydiff_score(c.d, p->dtype, K, c.ws, scores_out, true, c.st); };
    return run(Kind::compress, p, KVP_SCORER_KEYDIFF, 0, {K, V, K_out, V_out, idx_out, nullptr}, no_operands, score,
               workspace, workspace_bytes, stream);
}

// ---- StreamingLLM --------------------------------------------------------------------------------
int kvp_streaming_score(const kvp_problem* p, int32_t n_sink, void* scores_out,
                        kvp_stream_t stream) {
    Dims d;
    int rc = validate(p, &d, false);
    if (rc) return rc;
    if (!scores_out) return KVP_ERR_NULL_POINTER;
    if (n_sink < 0) return KVP_ERR_BAD_ARGUMENT;
    return status(launch_streaming_score(d, p->dtype, n_sink, scores_out, static_cast<cudaStream_t>(stream)));
}

int kvp_streaming_compress(const kvp_problem* p, int32_t n_sink, const void* K, const void* V,
                           void* K_out, void* V_out, int32_t* idx_out, kvp_stream_t stream) {
    Dims d;
    int rc = validate(p, &d);
    if (rc) return rc;
    if (n_sink < 0) return KVP_ERR_BAD_ARGUMENT;
    if (d.n_kept == 0) return KVP_OK;
    if ((rc = check_io(K, V, K_out, V_out))) return rc;
    return status(launch_streaming_compress(d, n_sink, K, V, K_out, V_out, idx_out, static_cast<cudaStream_t>(stream)));
}

// ---- SnapKV --------------------------------------------------------------------------------------
static int snapkv_window_ok(const Dims& d, int32_t window, int32_t kernel_size) {
    const bool ok = window > 0 && window < d.S && kernel_size > 0 && (kernel_size & 1) == 1;
    return ok ? KVP_OK : KVP_ERR_BAD_ARGUMENT;
}

static auto snapkv_stage(const kvp_problem* p, const void* K, const void* q_window, int32_t window,
                         int32_t kernel_size, void* scores_out) {
    return [=](const Call& c) {
        return launch_snapkv_score(c.d, p->dtype, K, q_window, window, kernel_size, c.ws, scores_out, c.st);
    };
}

int kvp_snapkv_score(const kvp_problem* p, const void* K, const void* q_window, int32_t window,
                     int32_t kernel_size, void* scores_out, void* workspace,
                     size_t workspace_bytes, kvp_stream_t stream) {
    auto operands = [&](const Dims& d) -> int {
        if (!K || !q_window || !scores_out) return KVP_ERR_NULL_POINTER;
        if (!aligned16(K) || !aligned16(q_window)) return KVP_ERR_BAD_STRIDE;
        return snapkv_window_ok(d, window, kernel_size);
    };
    return run(Kind::score, p, KVP_SCORER_SNAPKV, window, {}, operands,
               snapkv_stage(p, K, q_window, window, kernel_size, scores_out), workspace, workspace_bytes, stream);
}

int kvp_snapkv_compress(const kvp_problem* p, const void* K, const void* V,
                        const void* q_window, int32_t window, int32_t kernel_size, void* K_out,
                        void* V_out, int32_t* idx_out, void* scores_out, void* workspace,
                        size_t workspace_bytes, kvp_stream_t stream) {
    auto operands = [&](const Dims& d) -> int {
        if (!q_window) return KVP_ERR_NULL_POINTER;
        if (!aligned16(q_window)) return KVP_ERR_BAD_STRIDE;
        return snapkv_window_ok(d, window, kernel_size);
    };
    return run(Kind::compress, p, KVP_SCORER_SNAPKV, window, {K, V, K_out, V_out, idx_out, nullptr}, operands,
               snapkv_stage(p, K, q_window, window, kernel_size, scores_out), workspace, workspace_bytes, stream);
}

// ---- ExpectedAttention ---------------------------------------------------------------------------
static auto ea_stage(const kvp_problem* p, const void* K, const void* V, const void* mu, const void* cov,
                     float epsilon, int32_t n_sink, int32_t use_vnorm, void* scores_out) {
    return [=](const Call& c) {
        return launch_ea_score(c.d, p->dtype, K, V, mu, cov, epsilon, n_sink, use_vnorm, c.ws, scores_out, c.st);
    };
}

int kvp_expected_attention_score(const kvp_problem* p, const void* K, const void* V,
                                 const void* mu, const void* cov, float epsilon, int32_t n_sink,
                                 int32_t use_vnorm, void* scores_out, void* workspace,
                                 size_t workspace_bytes, kvp_stream_t stream) {
    auto operands = [&](const Dims& d) {
        if (!K || !mu || !scores_out || (use_vnorm && !V)) return KVP_ERR_NULL_POINTER;
        if (!aligned16(K) || !aligned16(mu) || (cov && !aligned16(cov))) return KVP_ERR_BAD_STRIDE;
        return (n_sink < 0 || n_sink >= d.S) ? KVP_ERR_BAD_ARGUMENT : KVP_OK;
    };
    return run(Kind::score, p, KVP_SCORER_EXPECTED_ATTENTION, 0, {}, operands,
               ea_stage(p, K, V, mu, cov, epsilon, n_sink, use_vnorm, scores_out), workspace, workspace_bytes, stream);
}

int kvp_expected_attention_compress(const kvp_problem* p, const void* K, const void* V,
                                    const void* mu, const void* cov, float epsilon,
                                    int32_t n_sink, int32_t use_vnorm, void* K_out, void* V_out,
                                    int32_t* idx_out, void* scores_out, void* workspace,
                                    size_t workspace_bytes, kvp_stream_t stream) {
    // V is checked with the other cache operands even when the score does not read it (use_vnorm == 0)
    auto operands = [&](const Dims& d) {
        if (!mu) return KVP_ERR_NULL_POINTER;
        if (!aligned16(mu) || (cov && !aligned16(cov))) return KVP_ERR_BAD_STRIDE;
        return (n_sink < 0 || n_sink >= d.S) ? KVP_ERR_BAD_ARGUMENT : KVP_OK;
    };
    return run(Kind::compress, p, KVP_SCORER_EXPECTED_ATTENTION, 0, {K, V, K_out, V_out, idx_out, nullptr}, operands,
               ea_stage(p, K, V, mu, cov, epsilon, n_sink, use_vnorm, scores_out), workspace, workspace_bytes, stream);
}

// ---- CriticalKV ----------------------------------------------------------------------------------
// The operand checks both entry points share, after their null / alignment checks; n_first_max is S for a score call,
// n_kept for a compress call.
static int criticalkv_args(const Dims& d, int32_t hidden, int64_t wo_stride, int32_t n_first, int32_t n_first_max) {
    if (hidden <= 0) return KVP_ERR_BAD_ARGUMENT;
    if (wo_stride % 8 != 0 || wo_stride < (int64_t)d.Hq * d.D) return KVP_ERR_BAD_STRIDE;
    return (n_first < 0 || n_first > n_first_max) ? KVP_ERR_BAD_ARGUMENT : KVP_OK;
}

static bool aligned2(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 1) == 0; }

int kvp_criticalkv_score(const kvp_problem* p, const void* V, const void* base_scores, const int64_t* score_stride,
                         const void* wo, int32_t hidden, int64_t wo_stride, float epsilon, int32_t n_first,
                         void* scores_out, void* workspace, size_t workspace_bytes, kvp_stream_t stream) {
    auto operands = [&](const Dims& d) -> int {
        if (!V || !base_scores || !score_stride || !wo || !scores_out) return KVP_ERR_NULL_POINTER;
        if (!aligned16(V) || !aligned2(base_scores) || !aligned16(wo)) return KVP_ERR_BAD_STRIDE;
        return criticalkv_args(d, hidden, wo_stride, n_first, d.S);
    };
    auto score = [&](const Call& c) {
        return launch_criticalkv_score(c.d, p->dtype, V, base_scores, score_stride[0], score_stride[1], wo, hidden,
                                       wo_stride, epsilon, n_first, c.ws, scores_out, c.st);
    };
    // the workspace is only read by the stage-1 selection
    return run(Kind::score, p, KVP_SCORER_CRITICALKV, 0, {}, operands, score, workspace, workspace_bytes, stream,
               n_first > 0);
}

int kvp_criticalkv_compress(const kvp_problem* p, const void* K, const void* V, const void* base_scores,
                            const int64_t* score_stride, const void* wo, int32_t hidden, int64_t wo_stride,
                            float epsilon, int32_t n_first, void* K_out, void* V_out, int32_t* idx_out,
                            void* scores_out, void* workspace, size_t workspace_bytes, kvp_stream_t stream) {
    auto operands = [&](const Dims& d) -> int {
        if (!base_scores || !score_stride || !wo) return KVP_ERR_NULL_POINTER;
        if (!aligned2(base_scores) || !aligned16(wo)) return KVP_ERR_BAD_STRIDE;
        return criticalkv_args(d, hidden, wo_stride, n_first, d.n_kept);
    };
    // the score stage, then the keys of the final scores for the selection: the stage-1 selection used the workspace
    auto score = [&](const Call& c) {
        void* out = scores_out ? scores_out : criticalkv_scratch_scores(c.d, c.ws);
        cudaError_t e = launch_criticalkv_score(c.d, p->dtype, V, base_scores, score_stride[0], score_stride[1], wo,
                                                hidden, wo_stride, epsilon, n_first, c.ws, out, c.st);
        if (e == cudaSuccess && n_first > 0) e = cudaMemsetAsync(c.ws.hist_hi, 0, c.zeroed, c.st);
        if (e == cudaSuccess)
            e = launch_keys_from_scores(c.d, p->dtype, out, (int64_t)c.d.H * c.d.S, c.d.S, c.ws, c.st);
        return e;
    };
    return run(Kind::compress, p, KVP_SCORER_CRITICALKV, 0, {K, V, K_out, V_out, idx_out, nullptr}, operands, score,
               workspace, workspace_bytes, stream);
}

// ---- ObservedAttention ---------------------------------------------------------------------------
// The operand checks both entry points share, after their null / alignment checks.
static int observed_attention_args(const Dims& d, int32_t n_q, float scaling) {
    if (n_q < 1 || n_q > d.S) return KVP_ERR_BAD_ARGUMENT;
    return (isfinite(scaling) && scaling > 0.f) ? KVP_OK : KVP_ERR_BAD_ARGUMENT;
}

static auto observed_attention_stage(const kvp_problem* p, const void* K, const void* q, int32_t n_q, float scaling,
                                     void* scores_out) {
    return [=](const Call& c) {
        return launch_observed_attention_score(c.d, p->dtype, K, q, n_q, scaling, c.ws, scores_out, c.st);
    };
}

int kvp_observed_attention_score(const kvp_problem* p, const void* K, const void* q, int32_t n_q, float scaling,
                                 void* scores_out, void* workspace, size_t workspace_bytes, kvp_stream_t stream) {
    auto operands = [&](const Dims& d) -> int {
        if (!K || !q || !scores_out) return KVP_ERR_NULL_POINTER;
        if (!aligned16(K) || !aligned16(q)) return KVP_ERR_BAD_STRIDE;
        return observed_attention_args(d, n_q, scaling);
    };
    return run(Kind::score, p, KVP_SCORER_OBSERVED_ATTENTION, n_q, {}, operands,
               observed_attention_stage(p, K, q, n_q, scaling, scores_out), workspace, workspace_bytes, stream);
}

int kvp_observed_attention_compress(const kvp_problem* p, const void* K, const void* V, const void* q, int32_t n_q,
                                    float scaling, void* K_out, void* V_out, int32_t* idx_out, void* scores_out,
                                    void* workspace, size_t workspace_bytes, kvp_stream_t stream) {
    auto operands = [&](const Dims& d) -> int {
        if (!q) return KVP_ERR_NULL_POINTER;
        if (!aligned16(q)) return KVP_ERR_BAD_STRIDE;
        return observed_attention_args(d, n_q, scaling);
    };
    return run(Kind::compress, p, KVP_SCORER_OBSERVED_ATTENTION, n_q, {K, V, K_out, V_out, idx_out, nullptr}, operands,
               observed_attention_stage(p, K, q, n_q, scaling, scores_out), workspace, workspace_bytes, stream);
}

// ---- NonCausalAttention --------------------------------------------------------------------------
// The operand checks both entry points share, after their null / alignment checks.
static int non_causal_attention_args(const Dims& d, int32_t chunk_size) {
    if (chunk_size < 1) return KVP_ERR_BAD_ARGUMENT;
    return non_causal_attention_supported(d, chunk_size) ? KVP_OK : KVP_ERR_UNSUPPORTED_SHAPE;
}

static auto non_causal_attention_stage(const kvp_problem* p, const void* K, const void* V, const void* q,
                                       int32_t chunk_size, void* scores_out) {
    return [=](const Call& c) {
        return launch_non_causal_attention_score(c.d, p->dtype, K, V, q, chunk_size, c.ws, scores_out, c.st);
    };
}

int kvp_non_causal_attention_score(const kvp_problem* p, const void* K, const void* V, const void* q,
                                   int32_t chunk_size, void* scores_out, void* workspace, size_t workspace_bytes,
                                   kvp_stream_t stream) {
    auto operands = [&](const Dims& d) -> int {
        if (!K || !V || !q || !scores_out) return KVP_ERR_NULL_POINTER;
        if (!aligned16(K) || !aligned16(V) || !aligned16(q)) return KVP_ERR_BAD_STRIDE;
        return non_causal_attention_args(d, chunk_size);
    };
    return run(Kind::score, p, KVP_SCORER_NON_CAUSAL_ATTENTION, 0, {}, operands,
               non_causal_attention_stage(p, K, V, q, chunk_size, scores_out), workspace, workspace_bytes, stream);
}

int kvp_non_causal_attention_compress(const kvp_problem* p, const void* K, const void* V, const void* q,
                                      int32_t chunk_size, void* K_out, void* V_out, int32_t* idx_out,
                                      void* scores_out, void* workspace, size_t workspace_bytes,
                                      kvp_stream_t stream) {
    auto operands = [&](const Dims& d) -> int {
        if (!q) return KVP_ERR_NULL_POINTER;
        if (!aligned16(q)) return KVP_ERR_BAD_STRIDE;
        return non_causal_attention_args(d, chunk_size);
    };
    return run(Kind::compress, p, KVP_SCORER_NON_CAUSAL_ATTENTION, 0, {K, V, K_out, V_out, idx_out, nullptr},
               operands, non_causal_attention_stage(p, K, V, q, chunk_size, scores_out), workspace, workspace_bytes,
               stream);
}

// ---- LagKV ---------------------------------------------------------------------------------------
// The operand checks both entry points share, after their null / alignment checks.
static int lagkv_args(int32_t n_sink, int32_t lag_size) {
    if (n_sink < 0 || lag_size < 1) return KVP_ERR_BAD_ARGUMENT;
    return lag_size > kLagMax ? KVP_ERR_UNSUPPORTED_SHAPE : KVP_OK;
}

int kvp_lagkv_score(const kvp_problem* p, const void* K, const void* V, int32_t n_sink, int32_t lag_size,
                    int32_t cross_scoring, void* scores_out, void* workspace, size_t workspace_bytes,
                    kvp_stream_t stream) {
    auto operands = [&](const Dims&) -> int {
        if (!K || !V || !scores_out) return KVP_ERR_NULL_POINTER;
        if (!aligned16(K) || !aligned16(V)) return KVP_ERR_BAD_STRIDE;
        return lagkv_args(n_sink, lag_size);
    };
    auto score = [&](const Call& c) {
        return launch_lagkv_score(c.d, p->dtype, K, V, n_sink, lag_size, cross_scoring, c.ws, scores_out, false, c.st);
    };
    // the kernel writes no keys and no histogram when the selection is skipped: nothing to clear
    return run(Kind::score, p, KVP_SCORER_LAGKV, 0, {}, operands, score, workspace, workspace_bytes, stream, false);
}

int kvp_lagkv_compress(const kvp_problem* p, const void* K, const void* V, int32_t n_sink, int32_t lag_size,
                       int32_t cross_scoring, void* K_out, void* V_out, int32_t* idx_out, void* scores_out,
                       void* workspace, size_t workspace_bytes, kvp_stream_t stream) {
    auto operands = [&](const Dims&) { return lagkv_args(n_sink, lag_size); };
    auto score = [&](const Call& c) {
        return launch_lagkv_score(c.d, p->dtype, K, V, n_sink, lag_size, cross_scoring, c.ws, scores_out, true, c.st);
    };
    return run(Kind::compress, p, KVP_SCORER_LAGKV, 0, {K, V, K_out, V_out, idx_out, nullptr}, operands, score,
               workspace, workspace_bytes, stream);
}

// ---- CUR -----------------------------------------------------------------------------------------
// The operand checks both entry points share, after their null / alignment checks.
static int cur_args(int32_t num_sinks, int32_t leverage_type, int32_t window, const float* G, int32_t r) {
    if (num_sinks < 0 || leverage_type < 0 || leverage_type > 3 || window < 0 || r < 0 || (G == nullptr) != (r == 0))
        return KVP_ERR_BAD_ARGUMENT;
    return (window > kCurWindowMax || r > kCurRankMax) ? KVP_ERR_UNSUPPORTED_SHAPE : KVP_OK;
}

static auto cur_stage(const kvp_problem* p, const void* K, const void* V, int32_t num_sinks, int32_t leverage_type,
                      int32_t window, const float* G, int32_t r, void* scores_out) {
    return [=](const Call& c) {
        return launch_cur_score(c.d, p->dtype, K, V, num_sinks, leverage_type, window, G, r, c.ws, scores_out, c.st);
    };
}

int kvp_cur_score(const kvp_problem* p, const void* K, const void* V, int32_t num_sinks, int32_t leverage_type,
                  int32_t local_window_size, const float* G, int32_t r, void* scores_out, void* workspace,
                  size_t workspace_bytes, kvp_stream_t stream) {
    auto operands = [&](const Dims&) -> int {
        if (!K || !V || !scores_out) return KVP_ERR_NULL_POINTER;
        if (!aligned16(K) || !aligned16(V)) return KVP_ERR_BAD_STRIDE;
        return cur_args(num_sinks, leverage_type, local_window_size, G, r);
    };
    return run(Kind::score, p, KVP_SCORER_CUR, 0, {}, operands,
               cur_stage(p, K, V, num_sinks, leverage_type, local_window_size, G, r, scores_out), workspace,
               workspace_bytes, stream);
}

int kvp_cur_compress(const kvp_problem* p, const void* K, const void* V, int32_t num_sinks, int32_t leverage_type,
                     int32_t local_window_size, const float* G, int32_t r, void* K_out, void* V_out, int32_t* idx_out,
                     void* scores_out, void* workspace, size_t workspace_bytes, kvp_stream_t stream) {
    auto operands = [&](const Dims&) { return cur_args(num_sinks, leverage_type, local_window_size, G, r); };
    return run(Kind::compress, p, KVP_SCORER_CUR, 0, {K, V, K_out, V_out, idx_out, nullptr}, operands,
               cur_stage(p, K, V, num_sinks, leverage_type, local_window_size, G, r, scores_out), workspace,
               workspace_bytes, stream);
}

// ---- generic scores ------------------------------------------------------------------------------
// The score stage of caller-supplied scores: their ordered keys and histogram.
static auto keys_from(const kvp_problem* p, const void* scores, const int64_t* score_stride) {
    return [=](const Call& c) {
        return launch_keys_from_scores(c.d, p->dtype, scores, score_stride[0], score_stride[1], c.ws, c.st);
    };
}

int kvp_scores_compress(const kvp_problem* p, const void* scores, const int64_t* score_stride,
                        const void* K, const void* V, void* K_out, void* V_out,
                        int32_t* idx_out, void* workspace, size_t workspace_bytes,
                        kvp_stream_t stream) {
    auto operands = [&](const Dims&) { return (!scores || !score_stride) ? KVP_ERR_NULL_POINTER : KVP_OK; };
    return run(Kind::compress, p, KVP_SCORER_GENERIC, 0, {K, V, K_out, V_out, idx_out, nullptr}, operands,
               keys_from(p, scores, score_stride), workspace, workspace_bytes, stream);
}

int kvp_scores_select(const kvp_problem* p, const void* scores, const int64_t* score_stride,
                      int32_t* idx_out, void* workspace, size_t workspace_bytes, kvp_stream_t stream) {
    auto operands = [&](const Dims&) { return (!scores || !score_stride || !idx_out) ? KVP_ERR_NULL_POINTER : KVP_OK; };
    return run(Kind::select, p, KVP_SCORER_GENERIC, 0, {nullptr, nullptr, nullptr, nullptr, idx_out, nullptr},
               operands, keys_from(p, scores, score_stride), workspace, workspace_bytes, stream);
}

int kvp_scores_compress_rerotate(const kvp_problem* p, const void* scores, const int64_t* score_stride,
                                 const void* K, const void* V, const float* inv_freq, void* K_out,
                                 void* V_out, int32_t* idx_out, void* workspace,
                                 size_t workspace_bytes, kvp_stream_t stream) {
    // rotate_half pairs d with d + D/2; checked ahead of the n_kept == 0 short cut
    Dims d;
    if (validate(p, &d) == KVP_OK && d.D % 16 != 0) return KVP_ERR_UNSUPPORTED_SHAPE;
    auto operands = [&](const Dims&) {
        return (!scores || !score_stride || !inv_freq) ? KVP_ERR_NULL_POINTER : KVP_OK;
    };
    return run(Kind::compress, p, KVP_SCORER_GENERIC, 0, {K, V, K_out, V_out, idx_out, inv_freq}, operands,
               keys_from(p, scores, score_stride), workspace, workspace_bytes, stream);
}

// ---- Merging -------------------------------------------------------------------------------------------------------
// The argument checks both entry points share, after their null / alignment checks. NaN fails every comparison.
static int merging_args(float similarity_threshold, double merge_fraction) {
    if (!(similarity_threshold >= 0.f && similarity_threshold <= 1.f)) return KVP_ERR_BAD_ARGUMENT;
    return (merge_fraction > 0.0 && merge_fraction <= 1.0) ? KVP_OK : KVP_ERR_BAD_ARGUMENT;
}

static bool aligned4(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3) == 0; }
static bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7) == 0; }
static size_t threshold_evict_workspace_bytes(int B, int Hkv, int n) {
    return align256((size_t)B * Hkv * ((n + kEvictTile - 1) / kEvictTile) * 8);
}

int kvp_merging_compress(const kvp_problem* p, const void* scores, const int64_t* score_stride, const void* K,
                         const void* V, float similarity_threshold, double merge_fraction, void* K_out, void* V_out,
                         int32_t* idx_out, int32_t* target_out, float* sim_out, void* workspace,
                         size_t workspace_bytes, kvp_stream_t stream) {
    auto operands = [&](const Dims&) -> int {
        if (!scores || !score_stride) return KVP_ERR_NULL_POINTER;
        if (!aligned4(target_out) || !aligned4(sim_out)) return KVP_ERR_BAD_STRIDE;
        return merging_args(similarity_threshold, merge_fraction);
    };
    // the merge rewrites the kept rows of V_out from V and the kept positions
    auto merge = [&](const Call& c, const int32_t* kept) {
        return launch_merging(c.d, p->dtype, K, V, kept, similarity_threshold, merge_fraction, V_out, target_out,
                              sim_out, c.ws, c.st);
    };
    const Io io = {K, V, K_out, V_out, idx_out, nullptr, merging_scratch_kept};
    return run(Kind::compress, p, KVP_SCORER_MERGING, 0, io, operands, keys_from(p, scores, score_stride), workspace,
               workspace_bytes, stream, true, merge);
}

int kvp_merging_merge(const kvp_problem* p, const void* K, const void* V, const int32_t* kept_idx,
                      float similarity_threshold, double merge_fraction, void* V_out, int32_t* target_out,
                      float* sim_out, void* workspace, size_t workspace_bytes, kvp_stream_t stream) {
    auto operands = [&](const Dims&) -> int {
        if (!K || !V || !kept_idx || !V_out) return KVP_ERR_NULL_POINTER;
        if (!aligned16(K) || !aligned16(V) || !aligned16(V_out) || !aligned4(kept_idx) || !aligned4(target_out) ||
            !aligned4(sim_out))
            return KVP_ERR_BAD_STRIDE;
        return merging_args(similarity_threshold, merge_fraction);
    };
    auto merge = [&](const Call& c) {
        return launch_merging(c.d, p->dtype, K, V, kept_idx, similarity_threshold, merge_fraction, V_out, target_out,
                              sim_out, c.ws, c.st);
    };
    // no selection: nothing to clear
    return run(Kind::score, p, KVP_SCORER_MERGING, 0, {}, operands, merge, workspace, workspace_bytes, stream, false);
}

// ---- ThinK ---------------------------------------------------------------------------------------------------------
kvp_status kvp_think_prune(const kvp_problem* p, void* K, const void* q_window, int32_t window, int32_t n_pruned,
                           int32_t* pruned_out, float* channel_scores_out, void* workspace, size_t workspace_bytes,
                           kvp_stream_t stream) {
    if (p == nullptr) return KVP_ERR_NULL_POINTER;
    kvp_problem pk = *p;  // V is not read: the problem is validated with K's strides in place of p->v_stride
    for (int i = 0; i < 3; ++i) pk.v_stride[i] = pk.k_stride[i];
    Call c;
    int rc = validate(&pk, &c.d);
    if (rc) return static_cast<kvp_status>(rc);
    if (window < 1 || n_pruned < 0 || n_pruned > c.d.D) return KVP_ERR_BAD_ARGUMENT;
    if (n_pruned == 0) return KVP_OK;
    if (!K || !q_window) return KVP_ERR_NULL_POINTER;
    if (!aligned16(K) || !aligned16(q_window) || !aligned4(pruned_out) || !aligned4(channel_scores_out))
        return KVP_ERR_BAD_STRIDE;
    c.st = static_cast<cudaStream_t>(stream);
    if ((rc = c.carve(KVP_SCORER_THINK, 0, workspace, workspace_bytes))) return static_cast<kvp_status>(rc);
    return static_cast<kvp_status>(status(launch_think_prune(c.d, p->dtype, K, q_window, window, n_pruned, pruned_out,
                                                             channel_scores_out, c.ws.scorer, c.st)));
}

// ---- Finch ---------------------------------------------------------------------------------------------------------
static auto finch_stage(const kvp_problem* p, const void* K, const void* q_window, int32_t window, int32_t normalize,
                        void* scores_out) {
    return [=](const Call& c) {
        return launch_finch_score(c.d, p->dtype, K, q_window, window, normalize, c.ws, scores_out, c.st);
    };
}

kvp_status kvp_finch_score(const kvp_problem* p, const void* K, const void* q_window, int32_t window, int32_t normalize,
                           void* scores_out, void* workspace, size_t workspace_bytes, kvp_stream_t stream) {
    auto operands = [&](const Dims& d) -> int {
        if (!K || !q_window || !scores_out) return KVP_ERR_NULL_POINTER;
        if (!aligned16(K) || !aligned16(q_window)) return KVP_ERR_BAD_STRIDE;
        int rc = finch_window_ok(d, window);
        return rc ? rc : finch_shape_ok(d);
    };
    return static_cast<kvp_status>(run(Kind::score, p, KVP_SCORER_FINCH, window, {}, operands,
                                       finch_stage(p, K, q_window, window, normalize, scores_out), workspace,
                                       workspace_bytes, stream));
}

kvp_status kvp_finch_compress(const kvp_problem* p, const void* K, const void* V, const void* q_window, int32_t window,
                              int32_t normalize, int32_t chunk_length, int32_t chunk_kept, int32_t tail_kept,
                              const float* inv_freq, void* K_out, void* V_out, int32_t* idx_out, void* scores_out,
                              void* workspace, size_t workspace_bytes, kvp_stream_t stream) {
    auto operands = [&](const Dims& d) -> int {
        if (!q_window) return KVP_ERR_NULL_POINTER;
        if (!aligned16(q_window)) return KVP_ERR_BAD_STRIDE;
        int rc = finch_window_ok(d, window);
        if (rc) return rc;
        if (chunk_length < 0) return KVP_ERR_BAD_ARGUMENT;
        if (chunk_length > 0 && (rc = chunk_counts_ok(d, chunk_length, chunk_kept, tail_kept))) return rc;
        return finch_shape_ok(d);
    };
    Io io = {K, V, K_out, V_out, idx_out, inv_freq};
    io.chunk_length = chunk_length;
    io.chunk_kept = chunk_kept;
    io.tail_kept = tail_kept;
    return static_cast<kvp_status>(run(Kind::compress, p, KVP_SCORER_FINCH, window, io, operands,
                                       finch_stage(p, K, q_window, window, normalize, scores_out), workspace,
                                       workspace_bytes, stream));
}

kvp_status kvp_scores_compress_chunked(const kvp_problem* p, const void* scores, const int64_t* score_stride,
                                       int32_t chunk_length, int32_t chunk_kept, int32_t tail_kept, const void* K,
                                       const void* V, const float* inv_freq, void* K_out, void* V_out,
                                       int32_t* idx_out, void* workspace, size_t workspace_bytes,
                                       kvp_stream_t stream) {
    auto operands = [&](const Dims& d) -> int {
        if (!scores || !score_stride) return KVP_ERR_NULL_POINTER;
        if (chunk_length < 1) return KVP_ERR_BAD_ARGUMENT;
        int rc = chunk_counts_ok(d, chunk_length, chunk_kept, tail_kept);
        if (rc) return rc;
        return inv_freq && d.D % 16 != 0 ? KVP_ERR_UNSUPPORTED_SHAPE : KVP_OK;
    };
    Io io = {K, V, K_out, V_out, idx_out, inv_freq};
    io.chunk_length = chunk_length;
    io.chunk_kept = chunk_kept;
    io.tail_kept = tail_kept;
    // the Finch layout at the smallest window: the selection regions and the kept positions
    return static_cast<kvp_status>(run(Kind::compress, p, KVP_SCORER_FINCH, 1, io, operands,
                                       keys_from(p, scores, score_stride), workspace, workspace_bytes, stream));
}

// ---- CaM -----------------------------------------------------------------------------------------------------------
kvp_status kvp_cam_compress(const kvp_problem* p, const void* scores, const int64_t* score_stride, const void* K,
                            const void* V, const float* attn_sum, const int64_t* attn_stride, int32_t n_merge,
                            int32_t merge_budget, const float* uniforms, void* K_out, void* V_out, float* attn_out,
                            const int64_t* attn_out_stride, int32_t* idx_out, int32_t* merge_idx_out,
                            float* merge_prob_out, void* workspace, size_t workspace_bytes, kvp_stream_t stream) {
    auto operands = [&](const Dims& d) -> int {
        if (!scores || !score_stride || !attn_sum || !attn_stride || !attn_out || !attn_out_stride)
            return KVP_ERR_NULL_POINTER;
        if (!uniforms && n_merge != 0) return KVP_ERR_NULL_POINTER;
        if (!aligned2(scores) || !aligned4(attn_sum) || !aligned4(attn_out) || !aligned4(uniforms) ||
            !aligned4(idx_out) || !aligned4(merge_idx_out) || !aligned4(merge_prob_out))
            return KVP_ERR_BAD_STRIDE;
        if (merge_budget < 1 || n_merge < 0 || n_merge > d.S - d.n_kept) return KVP_ERR_BAD_ARGUMENT;
        return KVP_OK;
    };
    Call c;
    int rc = prepare(Kind::compress, p, KVP_SCORER_CAM, 0, {K, V, K_out, V_out, idx_out, nullptr}, operands, workspace,
                     workspace_bytes, stream, &c);
    if (rc || c.d.n_kept == 0) return static_cast<kvp_status>(rc);
    if ((rc = c.zero())) return static_cast<kvp_status>(rc);
    return static_cast<kvp_status>(status(launch_cam_compress(
        c.d, p->dtype, scores, score_stride[0], score_stride[1], K, V, attn_sum, attn_stride[0], attn_stride[1],
        n_merge, merge_budget, uniforms, K_out, V_out, attn_out, attn_out_stride[0], attn_out_stride[1], idx_out,
        merge_idx_out, merge_prob_out, c.ws, c.st)));
}

// ---- KVzap ---------------------------------------------------------------------------------------------------------
// The operand checks both entry points share, after the problem's (see kvp_kvzap_score in the header).
static int kvzap_args(const Dims& d, const void* x, const int64_t* x_stride, int32_t hidden, int32_t hd,
                      const void* w1, const void* b1, const void* w2, const void* b2) {
    if (!x || !x_stride || !w1 || !b1 || (hd > 0 && (!w2 || !b2))) return KVP_ERR_NULL_POINTER;
    if (!aligned16(x) || !aligned16(w1) || !aligned2(b1) || !aligned2(w2) || !aligned2(b2)) return KVP_ERR_BAD_STRIDE;
    if (hidden < 1 || hd < 0) return KVP_ERR_BAD_ARGUMENT;
    for (int i = 0; i < 2; ++i)
        if (x_stride[i] < 0 || x_stride[i] % 8 != 0) return KVP_ERR_BAD_STRIDE;
    if (d.S > 1 && x_stride[1] < hidden) return KVP_ERR_BAD_STRIDE;
    if (hidden % 8 != 0 || hidden > kZapMaxHidden || hd % 8 != 0 || hd > kZapMaxHd || d.H > kZapMaxHeads)
        return KVP_ERR_UNSUPPORTED_SHAPE;
    return KVP_OK;
}

kvp_status kvp_kvzap_score(const kvp_problem* p, const void* x, const int64_t* x_stride, int32_t hidden, int32_t hd,
                           const void* w1, const void* b1, const void* w2, const void* b2, void* scores_out,
                           void* workspace, size_t workspace_bytes, kvp_stream_t stream) {
    auto operands = [&](const Dims& d) -> int {
        if (!scores_out) return KVP_ERR_NULL_POINTER;
        if (!aligned2(scores_out)) return KVP_ERR_BAD_STRIDE;
        return kvzap_args(d, x, x_stride, hidden, hd, w1, b1, w2, b2);
    };
    auto score = [&](const Call& c) {
        return launch_kvzap_score(c.d, p->dtype, x, x_stride[0], x_stride[1], hidden, hd, w1, b1, w2, b2, c.ws,
                                  scores_out, c.st);
    };
    // no selection: nothing to clear
    return static_cast<kvp_status>(run(Kind::score, p, KVP_SCORER_KVZAP, 0, {}, operands, score, workspace,
                                       workspace_bytes, stream, false));
}

kvp_status kvp_kvzap_compress(const kvp_problem* p, const void* x, const int64_t* x_stride, int32_t hidden, int32_t hd,
                              const void* w1, const void* b1, const void* w2, const void* b2, const void* K,
                              const void* V, void* K_out, void* V_out, int32_t* idx_out, void* scores_out,
                              void* workspace, size_t workspace_bytes, kvp_stream_t stream) {
    auto operands = [&](const Dims& d) -> int {
        if (!aligned2(scores_out)) return KVP_ERR_BAD_STRIDE;
        return kvzap_args(d, x, x_stride, hidden, hd, w1, b1, w2, b2);
    };
    auto score = [&](const Call& c) {
        void* out = scores_out ? scores_out : kvzap_scratch_scores(c.d, c.ws);
        cudaError_t e = launch_kvzap_score(c.d, p->dtype, x, x_stride[0], x_stride[1], hidden, hd, w1, b1, w2, b2,
                                           c.ws, out, c.st);
        if (e == cudaSuccess)
            e = launch_keys_from_scores(c.d, p->dtype, out, (int64_t)c.d.H * c.d.S, c.d.S, c.ws, c.st);
        return e;
    };
    return static_cast<kvp_status>(run(Kind::compress, p, KVP_SCORER_KVZAP, 0, {K, V, K_out, V_out, idx_out, nullptr},
                                       operands, score, workspace, workspace_bytes, stream));
}

// ---- DMS threshold eviction -----------------------------------------------------------------------------------------
kvp_status kvp_threshold_evict(int32_t dtype, int32_t B, int32_t Hkv, int32_t n, const void* scores,
                               const int64_t* score_stride, int32_t n_evict, float threshold, int64_t shift,
                               int64_t* b_out, int64_t* h_out, int64_t* s_out, int64_t* count_out, void* workspace,
                               size_t workspace_bytes, kvp_stream_t stream) {
    if (dtype != KVP_BF16 && dtype != KVP_F16) return KVP_ERR_UNSUPPORTED_DTYPE;
    // one CTA per (row, tile of kEvictTile positions) on gridDim.x
    if (B <= 0 || Hkv <= 0 || n <= 0 || (int64_t)B * Hkv * ((n + kEvictTile - 1) / kEvictTile) > 0x7FFFFFFF)
        return KVP_ERR_UNSUPPORTED_SHAPE;
    if (n_evict < 0 || n_evict > n) return KVP_ERR_BAD_ARGUMENT;
    if (!scores || !score_stride || !count_out || (n_evict > 0 && (!b_out || !h_out || !s_out)))
        return KVP_ERR_NULL_POINTER;
    if (!aligned2(scores) || score_stride[0] < 0 || score_stride[1] < 0 || !aligned8(b_out) || !aligned8(h_out) ||
        !aligned8(s_out) || !aligned8(count_out))
        return KVP_ERR_BAD_STRIDE;
    if (workspace == nullptr) return KVP_ERR_NULL_POINTER;
    if (!aligned16(workspace)) return KVP_ERR_BAD_STRIDE;
    if (workspace_bytes < threshold_evict_workspace_bytes(B, Hkv, n)) return KVP_ERR_WORKSPACE_TOO_SMALL;
    return static_cast<kvp_status>(status(launch_threshold_evict(dtype, B, Hkv, scores, score_stride[0],
                                                                 score_stride[1], n_evict, threshold, shift, b_out,
                                                                 h_out, s_out, count_out, workspace,
                                                                 static_cast<cudaStream_t>(stream))));
}

}  // extern "C"
