// Final RMSNorm + lm_head + greedy argmax for decode-shaped inputs (M <= 8 rows).
// logits are produced by the weight-streaming GEMV (bf16, as the reference's lm_head emits them), then a
// two-stage argmax picks the lowest index among equal maxima, which is what torch.argmax returns.
// With PROC the argmax runs over HF's processed values (repetition penalty, ban set: logits_process.cu), computed in
// fp32 as each logit is read, and the final stage appends the picked id to the row's history.
// With LOG the part kernel also stores every value it reads into the score log (common.cuh LogDesc): nothing else reads
// the row again.
#include "common.cuh"

namespace tl {

constexpr int AM_PARTS = 64, AM_THREADS = 256;

template <bool PROC, bool LOG = false>
__global__ void __launch_bounds__(AM_THREADS) argmax_part_kernel(const bf16* __restrict__ logits, float* __restrict__ pval,
                                                                 int* __restrict__ pidx, int V, LpRows h, LogDesc lg) {
    const int m = blockIdx.y, part = blockIdx.x;
    const int per = (V + AM_PARTS - 1) / AM_PARTS;
    const int lo = part * per, hi = min(V, lo + per);
    const bf16* row = logits + (size_t)m * V;
    const uint32_t* bits = PROC ? h.bits + (size_t)m * h.W : nullptr;
    const uint32_t* ban = PROC && h.ban ? h.ban + (size_t)m * h.W : nullptr;
    const float penalty = PROC ? __int_as_float(h.params[TL_LP_PENALTY]) : 1.f;
    float *raw = nullptr, *proc = nullptr;
    const bool log = LOG && log_rows(lg, *lg.col, m, V, &raw, &proc);
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = lo + threadIdx.x; i < hi; i += AM_THREADS) {
        const float x = bf2f(row[i]);
        float v = x;
        if (PROC) v = lp_value(v, i, bits, ban, penalty);
        if (LOG && log) {                       // greedy: the score is the processed value (the logit itself without PROC)
            if (raw) raw[i] = x;
            if (proc) proc[i] = v;
        }
        if (v > best) { best = v; bi = i; }     // ascending i per thread: first max kept
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    __shared__ float sv[AM_THREADS / 32];
    __shared__ int si[AM_THREADS / 32];
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best; si[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < AM_THREADS / 32; ++w)
            if (sv[w] > best || (sv[w] == best && si[w] < bi)) { best = sv[w]; bi = si[w]; }
        pval[m * AM_PARTS + part] = best;
        pidx[m * AM_PARTS + part] = bi;
    }
}

// LOG: the step's last kernel advances the log column, after every part kernel read it (stream order)
template <bool PROC, bool LOG = false>
__global__ void argmax_final_kernel(const float* __restrict__ pval, const int* __restrict__ pidx,
                                    int64_t* __restrict__ ids_out, LpRows h, int32_t* __restrict__ log_col) {
    const int m = blockIdx.x, lane = threadIdx.x;
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = lane; i < AM_PARTS; i += 32) {
        const float v = pval[m * AM_PARTS + i];
        const int ix = pidx[m * AM_PARTS + i];
        if (v > best || (v == best && ix < bi)) { best = v; bi = ix; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if (lane == 0) {
        const int id = (bi == 0x7fffffff) ? 0 : bi;
        ids_out[m] = (int64_t)id;
        if (PROC) lp_append(h, m, id);
        if (LOG && m == 0) log_col[0] += 1;
    }
}

}  // namespace tl

extern "C" {

size_t tl_lmhead_ws(int M, int V) {
    return (size_t)M * V * sizeof(tl::bf16) + (size_t)M * tl::AM_PARTS * (sizeof(float) + sizeof(int)) + 256;
}

static int argmax_launch(const void* logits, int64_t* ids_out, void* workspace, size_t ws_bytes, int M, int V, const tl::LogDesc* lg,
                         void* stream) {
    using namespace tl;
    const size_t need = (size_t)M * AM_PARTS * (sizeof(float) + sizeof(int));
    TL_REQUIRE(ws_bytes >= need, TL_ERR_WORKSPACE, "tl_argmax_bf16: workspace %zu < %zu", ws_bytes, need);
    if (M == 0) return TL_OK;
    float* pval = (float*)workspace;
    int* pidx = (int*)(pval + (size_t)M * AM_PARTS);
    cudaStream_t st = (cudaStream_t)stream;
    if (lg) {
        argmax_part_kernel<false, true><<<dim3(AM_PARTS, M), AM_THREADS, 0, st>>>((const bf16*)logits, pval, pidx, V, LpRows{}, *lg);
        argmax_final_kernel<false, true><<<M, 32, 0, st>>>(pval, pidx, ids_out, LpRows{}, lg->col);
    } else {
        argmax_part_kernel<false><<<dim3(AM_PARTS, M), AM_THREADS, 0, st>>>((const bf16*)logits, pval, pidx, V, LpRows{}, LogDesc{});
        argmax_final_kernel<false><<<M, 32, 0, st>>>(pval, pidx, ids_out, LpRows{}, nullptr);
    }
    return check_launch("tl_argmax_bf16");
}

int tl_argmax_bf16(const void* logits, int64_t* ids_out, void* workspace, size_t ws_bytes, int M, int V, void* stream) {
    return argmax_launch(logits, ids_out, workspace, ws_bytes, M, V, nullptr, stream);
}

int tl_argmax_bf16_log(const void* logits, int64_t* ids_out, void* workspace, size_t ws_bytes, int M, int V, float* raw_log,
                       float* score_log, int32_t* log_col, int n_cols, int B_total, int row0, void* stream) {
    using namespace tl;
    TL_REQUIRE(logits && ids_out && workspace, TL_ERR_INVALID, "tl_argmax_bf16_log: null argument");
    LogDesc lg;
    const int rc = make_log("tl_argmax_bf16_log", raw_log, score_log, log_col, n_cols, B_total, row0, M, V, 1.f, &lg);
    if (rc != TL_OK) return rc;
    return argmax_launch(logits, ids_out, workspace, ws_bytes, M, V, &lg, stream);
}

static int argmax_proc_launch(const void* logits, int64_t* ids_out, int32_t* log, int32_t* len, uint32_t* bits,
                              const int32_t* params_dev, int flags, void* workspace, size_t ws_bytes, int M, int V, int L,
                              const tl::LogDesc* lg, void* stream) {
    using namespace tl;
    TL_REQUIRE(logits && ids_out && log && len && bits && params_dev && workspace, TL_ERR_INVALID, "tl_argmax_proc: null argument");
    TL_REQUIRE(M >= 1 && V >= 1 && L >= 1, TL_ERR_INVALID, "tl_argmax_proc: bad shape M=%d V=%d L=%d", M, V, L);
    TL_REQUIRE(ws_bytes >= tl_logits_proc_ws(M, V), TL_ERR_WORKSPACE, "tl_argmax_proc: workspace %zu < %zu", ws_bytes,
               tl_logits_proc_ws(M, V));
    cudaStream_t st = (cudaStream_t)stream;
    uint32_t* ban = (uint32_t*)workspace;
    float* pval = (float*)((unsigned char*)workspace + lp_ban_bytes(M, V));
    int* pidx = (int*)(pval + (size_t)M * AM_PARTS);
    const LpRows h{log, len, bits, (flags & TL_LP_BAN) ? ban : nullptr, params_dev, L, lp_words(V)};
    if (flags & TL_LP_BAN) {
        const int rc = lp_ban_launch(h, ban, M, V, st);
        if (rc != TL_OK) return rc;
    }
    if (lg) {
        argmax_part_kernel<true, true><<<dim3(AM_PARTS, M), AM_THREADS, 0, st>>>((const bf16*)logits, pval, pidx, V, h, *lg);
        argmax_final_kernel<true, true><<<M, 32, 0, st>>>(pval, pidx, ids_out, h, lg->col);
    } else {
        argmax_part_kernel<true><<<dim3(AM_PARTS, M), AM_THREADS, 0, st>>>((const bf16*)logits, pval, pidx, V, h, LogDesc{});
        argmax_final_kernel<true><<<M, 32, 0, st>>>(pval, pidx, ids_out, h, nullptr);
    }
    return check_launch("tl_argmax_proc");
}

int tl_argmax_proc(const void* logits, int64_t* ids_out, int32_t* log, int32_t* len, uint32_t* bits,
                   const int32_t* params_dev, int flags, void* workspace, size_t ws_bytes, int M, int V, int L, void* stream) {
    return argmax_proc_launch(logits, ids_out, log, len, bits, params_dev, flags, workspace, ws_bytes, M, V, L, nullptr, stream);
}

int tl_argmax_proc_log(const void* logits, int64_t* ids_out, int32_t* log, int32_t* len, uint32_t* bits,
                       const int32_t* params_dev, int flags, void* workspace, size_t ws_bytes, int M, int V, int L,
                       float* raw_log, float* score_log, int32_t* log_col, int n_cols, int B_total, int row0, void* stream) {
    using namespace tl;
    LogDesc lg;
    const int rc = make_log("tl_argmax_proc_log", raw_log, score_log, log_col, n_cols, B_total, row0, M, V, 1.f, &lg);
    if (rc != TL_OK) return rc;
    return argmax_proc_launch(logits, ids_out, log, len, bits, params_dev, flags, workspace, ws_bytes, M, V, L, &lg, stream);
}

int tl_lmhead_argmax(const void* x, const void* W, const void* norm_w, float eps, int64_t* ids_out, void* logits_out,
                     void* workspace, size_t ws_bytes, int M, int V, int H, unsigned* gemv_counter, void* stream) {
    using namespace tl;
    TL_REQUIRE(M >= 1 && M <= 8, TL_ERR_INVALID, "tl_lmhead_argmax: M=%d outside 1..8", M);
    TL_REQUIRE(ws_bytes >= tl_lmhead_ws(M, V), TL_ERR_WORKSPACE, "tl_lmhead_argmax: workspace %zu < %zu", ws_bytes,
               tl_lmhead_ws(M, V));
    unsigned char* ws = (unsigned char*)workspace;
    void* logits = logits_out ? logits_out : (void*)ws;
    size_t off = ((size_t)M * V * sizeof(bf16) + 255) & ~(size_t)255;
    int rc = tl_gemv_bf16_ctr(x, W, logits, M, V, H, nullptr, nullptr, norm_w, eps, 0, gemv_counter, nullptr, 0, stream);
    if (rc != TL_OK) return rc;
    return tl_argmax_bf16(logits, ids_out, ws + off, ws_bytes - off, M, V, stream);
}

}  // extern "C"
