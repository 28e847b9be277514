// Shared device/host helpers for the tensorlink_b200 sm_90a kernels.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/tensorlink_b200.h"

namespace tl {

typedef __nv_bfloat16 bf16;

// ---------------------------------------------------------------- host-side error plumbing
void set_error(const char* fmt, ...);
int check_launch(const char* what);   // cudaGetLastError -> TL_ERR_CUDA + message

#define TL_REQUIRE(cond, code, ...)                \
    do {                                           \
        if (!(cond)) {                             \
            tl::set_error(__VA_ARGS__);            \
            return (code);                         \
        }                                          \
    } while (0)

int sm_count();

// ---------------------------------------------------------------- bf16 helpers (exact HF rounding points)
__device__ __forceinline__ float bf2f(bf16 v) { return __bfloat162float(v); }
__device__ __forceinline__ bf16 f2bf(float v) { return __float2bfloat16_rn(v); }
// round-trip: the value a bf16 tensor would hold
__device__ __forceinline__ float rbf(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

__device__ __forceinline__ float bf16_lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t u) { return __uint_as_float(u & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
    __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&t);
}
// torch CPU: silu on a bf16 tensor = fp32 x/(1+exp(-x)) rounded to bf16.  The fp32 value only has to be right to
// well under a bf16 ulp (2^-9), so the SFU forms are used: the IEEE division + expf pair is a long dependent chain
// per element in the GEMM epilogue.
__device__ __forceinline__ float silu_f(float x) { return x * __frcp_rn(1.0f + __expf(-x)); }

__device__ __forceinline__ uint4 ldg_nc_v4(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// ---------------------------------------------------------------- logits processors (csrc/logits_process.cu)
// One row's token history (log, length, presence bitmap) and the parameters, as tl_argmax_proc / tl_sample_proc get them.
struct LpRows {
    int32_t* log;               // [M, L]
    int32_t* len;               // [M]
    uint32_t* bits;             // [M, W]: bit v set = token v is in the history
    const uint32_t* ban;        // [M, W] ban set of this step, or nullptr
    const int32_t* params;      // TL_LP_* layout (include/tensorlink_b200.h)
    int L, W;
};
__host__ __device__ __forceinline__ int lp_words(int V) { return (V + 31) / 32; }
inline size_t lp_ban_bytes(int M, int V) { return ((size_t)M * lp_words(V) * sizeof(uint32_t) + 255) & ~(size_t)255; }
// HF RepetitionPenaltyLogitsProcessor on the fp32 copy of a logit, then the ban set (-inf)
__device__ __forceinline__ float lp_value(float s, int i, const uint32_t* bits, const uint32_t* ban, float penalty) {
    if (ban && ((ban[i >> 5] >> (i & 31)) & 1u)) return -INFINITY;
    if ((bits[i >> 5] >> (i & 31)) & 1u) s = s < 0.f ? __fmul_rn(s, penalty) : __fdiv_rn(s, penalty);
    return s;
}
// the picked token joins row m's history (one thread per row)
__device__ __forceinline__ void lp_append(const LpRows& h, int m, int id) {
    const int n = h.len[m];
    if (n < h.L) h.log[(size_t)m * h.L + n] = id;
    h.len[m] = n + 1;
    h.bits[(size_t)m * h.W + (id >> 5)] |= 1u << (id & 31);
}
// the ban set of every row into h.ban (the first lp_ban_bytes(M, V) of the workspace): n-gram completions and the EOS
// ids while below min_new_tokens
int lp_ban_launch(const LpRows& h, uint32_t* ban, int M, int V, cudaStream_t stream);

// ---------------------------------------------------------------- score log (generate's output_scores / output_logits)
// The picking kernels of a decode step (the argmax, the samplers) also store each row's values into column c of fp32
// logs [n_cols, B_total, V]: raw = float(bf16 logit) and proc = the score HF returns (processed, warped).  c is read from
// device memory and the step's last kernel advances it, so a captured graph writes every replay into the next column.
struct LogDesc {
    float* raw;                 // or nullptr
    float* proc;                // or nullptr
    int32_t* col;               // {column, exit word}: the exit word is zero between launches (last_cta_out)
    long long col_stride;       // B_total * V
    int row0, n_cols;           // row m of the launch is log row row0 + m; columns >= n_cols are not written
    float temperature;          // the samplers' score of a kept value x: x / temperature (IEEE division, as HF)
};
// the log rows of launch row m in column c, or false when c lies outside the log
__device__ __forceinline__ bool log_rows(const LogDesc& d, int c, int m, int V, float** raw, float** proc) {
    if (c < 0 || c >= d.n_cols) return false;
    const long long off = (long long)c * d.col_stride + (long long)(d.row0 + m) * V;
    *raw = d.raw ? d.raw + off : nullptr;
    *proc = d.proc ? d.proc + off : nullptr;
    return true;
}
// checks a log's arguments for M rows of V values and fills *d (the host half of every _log entry point)
inline int make_log(const char* who, float* raw, float* proc, int32_t* col, int n_cols, int B_total, int row0, int M, int V,
                    float temperature, LogDesc* d) {
    TL_REQUIRE(col, TL_ERR_INVALID, "%s: null column counter", who);
    TL_REQUIRE(raw || proc, TL_ERR_INVALID, "%s: neither a raw nor a score log", who);
    TL_REQUIRE(n_cols >= 1 && row0 >= 0 && M >= 0 && V >= 1 && (long long)row0 + M <= B_total, TL_ERR_INVALID,
               "%s: bad log shape n_cols=%d B_total=%d row0=%d M=%d", who, n_cols, B_total, row0, M);
    const long long stride = (long long)B_total * V;
    TL_REQUIRE(stride <= (long long)(~0ull >> 1) / n_cols, TL_ERR_INVALID, "%s: a log of %d x %d x %d values overflows",
               who, n_cols, B_total, V);
    *d = LogDesc{raw, proc, col, stride, row0, n_cols, temperature};
    return TL_OK;
}

// ---------------------------------------------------------------- mbarrier / TMA PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {}
}

__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
// 2-D tiled load global -> shared, completion on an mbarrier (transaction bytes)
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
// 1-D bulk copy global -> shared (no tensor map), completion on an mbarrier
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// ---------------------------------------------------------------- work tickets
// A launch hands out its work units in address order from a device counter: a CTA takes n consecutive units at a time,
// so an SM that streams faster simply takes more and all CTAs finish within one ticket of each other.  The counter
// words are zero when a launch starts and the last CTA out leaves them zero, so a launch must never share them with
// another launch that can run at the same time.
__device__ __forceinline__ int ticket_take(unsigned* ctr, int n) { return (int)atomicAdd(ctr, (unsigned)n); }
// Called once per CTA, after the CTA's last use of the launch's counters.  True in exactly one CTA, the last to get
// here, which has already zeroed `exit_word` and must zero the other counters (then __threadfence()).
__device__ __forceinline__ bool last_cta_out(unsigned* exit_word) {
    __threadfence();                       // this thread's counter atomics are performed before its exit is counted
    if (atomicAdd(exit_word, 1u) != gridDim.x - 1) return false;
    *exit_word = 0u;
    return true;
}

}  // namespace tl
