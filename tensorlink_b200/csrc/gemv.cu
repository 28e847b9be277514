// Decode-shaped Linear: y[M,N] = f(norm(x)[M,K] · W[N,K]^T), M <= 8.  HBM-bound weight streaming.
//
// Work item = G consecutive row PAIRS of W (a pair is gate/up for the SwiGLU epilogue).  WPI warps share
// an item and split K between them with a CTA-coalesced stride; 8/WPI items are in flight per CTA.
// Every lane keeps 2*G independent 16-byte loads in flight per k-iteration (ld.global.nc, L1 no-allocate).
// Algorithmic bytes per launch = 2*N*K (weights) + O(M*(K+N)) activations.
#include <stdlib.h>

#include <atomic>
#include <mutex>

#include "common.cuh"
#include "fp8.cuh"

namespace tl {

constexpr int GEMV_THREADS = 256;
constexpr int GEMV_WARPS = GEMV_THREADS / 32;

// The body of both kernels below.  WT: bf16, or fp8_e4m3 with `scales` [N][K/128]: each lane forms bf16(float(w) *
// scale) from an 8-byte vector at the bf16 kernel's vector index, so the FMA sequence of every output is the bf16
// kernel's over the dequantized matrix.
template <typename WT, int M, int G, int WPI>
__device__ __forceinline__ void gemv_body(const bf16* __restrict__ x, const WT* __restrict__ W, bf16* __restrict__ y,
                                          int N, int K, const bf16* __restrict__ bias, const bf16* __restrict__ residual,
                                          const bf16* __restrict__ norm_w, float eps, int flags,
                                          const float* __restrict__ scales) {
    constexpr bool FP8 = sizeof(WT) == 1;
    constexpr int SLOTS = GEMV_WARPS / WPI;
    constexpr int ROWS = 2 * G;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    bf16* xs = reinterpret_cast<bf16*>(smem_raw);                                  // [M][K]
    float* red = reinterpret_cast<float*>(smem_raw + (size_t)M * K * sizeof(bf16));  // [WARPS][ROWS*M]
    __shared__ float s_part[GEMV_WARPS][M];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nvec = K >> 3;

    // ---- prologue: stage x (optionally RMS-normalised with HF rounding) in shared memory
    if (norm_w) {
        float ss[M];
#pragma unroll
        for (int m = 0; m < M; ++m) ss[m] = 0.f;
        for (int v = tid; v < nvec; v += GEMV_THREADS) {
#pragma unroll
            for (int m = 0; m < M; ++m) {
                uint4 u = reinterpret_cast<const uint4*>(x + (size_t)m * K)[v];
                const uint32_t* w32 = reinterpret_cast<const uint32_t*>(&u);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    float a = bf16_lo(w32[j]), b = bf16_hi(w32[j]);
                    ss[m] += a * a + b * b;
                }
            }
        }
#pragma unroll
        for (int m = 0; m < M; ++m) {
            float t = warp_sum(ss[m]);
            if (lane == 0) s_part[warp][m] = t;
        }
        __syncthreads();
        float rstd[M];
#pragma unroll
        for (int m = 0; m < M; ++m) {
            float t = 0.f;
#pragma unroll
            for (int w = 0; w < GEMV_WARPS; ++w) t += s_part[w][m];
            rstd[m] = 1.0f / sqrtf(t / (float)K + eps);
        }
        for (int v = tid; v < nvec; v += GEMV_THREADS) {
            uint4 g = reinterpret_cast<const uint4*>(norm_w)[v];
            const uint32_t* g32 = reinterpret_cast<const uint32_t*>(&g);
#pragma unroll
            for (int m = 0; m < M; ++m) {
                uint4 u = reinterpret_cast<const uint4*>(x + (size_t)m * K)[v], o;
                const uint32_t* u32 = reinterpret_cast<const uint32_t*>(&u);
                uint32_t* o32 = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    o32[j] = pack_bf16(bf16_lo(g32[j]) * rbf(bf16_lo(u32[j]) * rstd[m]),
                                       bf16_hi(g32[j]) * rbf(bf16_hi(u32[j]) * rstd[m]));
                reinterpret_cast<uint4*>(xs + (size_t)m * K)[v] = o;
            }
        }
    } else {
        for (int v = tid; v < nvec * M; v += GEMV_THREADS)
            reinterpret_cast<uint4*>(xs)[v] = reinterpret_cast<const uint4*>(x)[v];
    }
    __syncthreads();

    const int npairs = N >> 1;
    const int n_items = (npairs + G - 1) / G;
    const int slot = warp / WPI, wi = warp % WPI;
    const bool swiglu = flags & TL_EPI_SWIGLU;
    const int n_out = swiglu ? npairs : N;

    for (int base = blockIdx.x * SLOTS; base < n_items; base += gridDim.x * SLOTS) {
        const int item = base + slot;
        float acc[ROWS][M];
#pragma unroll
        for (int r = 0; r < ROWS; ++r)
#pragma unroll
            for (int m = 0; m < M; ++m) acc[r][m] = 0.f;
        if (item < n_items) {
            const int row0 = item * ROWS;
            const WT* wrow[ROWS];
            const float* srow[ROWS];
#pragma unroll
            for (int r = 0; r < ROWS; ++r) {
                int row = row0 + r;
                if (row >= N) row = N - 1;   // clamp (result discarded)
                wrow[r] = W + (size_t)row * K;
                if constexpr (FP8) srow[r] = scales + (size_t)row * (K / TL_FP8_BLOCK);
            }
#pragma unroll 2
            for (int v = wi * 32 + lane; v < nvec; v += WPI * 32) {
                uint4 wv[ROWS];
                float wf[FP8 ? ROWS : 1][8];
#pragma unroll
                for (int r = 0; r < ROWS; ++r) {
                    if constexpr (FP8)
                        fp8x8_scaled(__ldg(reinterpret_cast<const uint2*>(wrow[r]) + v), __ldg(srow[r] + (v >> 4)), wf[r]);
                    else
                        wv[r] = ldg_nc_v4(reinterpret_cast<const uint4*>(wrow[r]) + v);
                }
#pragma unroll
                for (int m = 0; m < M; ++m) {
                    const uint4 xv = reinterpret_cast<const uint4*>(xs + (size_t)m * K)[v];
                    const uint32_t* x32 = reinterpret_cast<const uint32_t*>(&xv);
                    float xf[8];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        xf[2 * j] = bf16_lo(x32[j]);
                        xf[2 * j + 1] = bf16_hi(x32[j]);
                    }
#pragma unroll
                    for (int r = 0; r < ROWS; ++r) {
                        if constexpr (FP8) {
#pragma unroll
                            for (int j = 0; j < 8; ++j) acc[r][m] = fmaf(wf[r][j], xf[j], acc[r][m]);
                        } else {
                            const uint32_t* w32 = reinterpret_cast<const uint32_t*>(&wv[r]);
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                acc[r][m] = fmaf(bf16_lo(w32[j]), xf[2 * j], acc[r][m]);
                                acc[r][m] = fmaf(bf16_hi(w32[j]), xf[2 * j + 1], acc[r][m]);
                            }
                        }
                    }
                }
            }
        }
#pragma unroll
        for (int r = 0; r < ROWS; ++r)
#pragma unroll
            for (int m = 0; m < M; ++m) {
                float t = warp_sum(acc[r][m]);
                if (lane == 0) red[warp * (ROWS * M) + r * M + m] = t;
            }
        __syncthreads();
        // ---- epilogue: one thread per (slot, pair g, token m)
        if (tid < SLOTS * G * M) {
            const int s = tid / (G * M), rem = tid - s * (G * M);
            const int g = rem / M, m = rem - g * M;
            const int it = base + s;
            const int r0 = (it * G + g) * 2;
            if (it < n_items && r0 < N) {
                float v0 = 0.f, v1 = 0.f;
#pragma unroll
                for (int w = 0; w < WPI; ++w) {
                    v0 += red[(s * WPI + w) * (ROWS * M) + (2 * g) * M + m];
                    v1 += red[(s * WPI + w) * (ROWS * M) + (2 * g + 1) * M + m];
                }
                if (flags & TL_EPI_BIAS) {
                    v0 += bf2f(bias[r0]);
                    v1 += bf2f(bias[r0 + 1]);
                }
                if (swiglu) {
                    const float gate = rbf(v0), up = rbf(v1);
                    y[(size_t)m * n_out + (r0 >> 1)] = f2bf(rbf(silu_f(gate)) * up);
                } else {
                    float t0 = rbf(v0), t1 = rbf(v1);
                    if (flags & TL_EPI_RESIDUAL) {
                        t0 += bf2f(residual[(size_t)m * N + r0]);
                        t1 += bf2f(residual[(size_t)m * N + r0 + 1]);
                    }
                    y[(size_t)m * N + r0] = f2bf(t0);
                    if (r0 + 1 < N) y[(size_t)m * N + r0 + 1] = f2bf(t1);
                }
            }
        }
        __syncthreads();
    }
}

template <int M, int G, int WPI>
__global__ void __launch_bounds__(GEMV_THREADS) gemv_kernel(const bf16* __restrict__ x, const bf16* __restrict__ W,
                                                            bf16* __restrict__ y, int N, int K,
                                                            const bf16* __restrict__ bias,
                                                            const bf16* __restrict__ residual,
                                                            const bf16* __restrict__ norm_w, float eps, int flags) {
    gemv_body<bf16, M, G, WPI>(x, W, y, N, K, bias, residual, norm_w, eps, flags, nullptr);
}

template <int M, int G, int WPI>
__global__ void __launch_bounds__(GEMV_THREADS) gemv_fp8_kernel(const bf16* __restrict__ x,
                                                                const fp8_e4m3* __restrict__ W, bf16* __restrict__ y,
                                                                int N, int K, const bf16* __restrict__ bias,
                                                                const bf16* __restrict__ residual,
                                                                const bf16* __restrict__ norm_w, float eps, int flags,
                                                                const float* __restrict__ scales) {
    gemv_body<fp8_e4m3, M, G, WPI>(x, W, y, N, K, bias, residual, norm_w, eps, flags, scales);
}

template <typename WT, int M, int G, int WPI>
static int launch_gemv(const void* x, const void* W, const float* scales, void* y, int N, int K, const void* bias,
                       const void* residual, const void* norm_w, float eps, int flags, cudaStream_t st) {
    constexpr int SLOTS = GEMV_WARPS / WPI;
    constexpr bool FP8 = sizeof(WT) == 1;
    const void* kern = FP8 ? (const void*)gemv_fp8_kernel<M, G, WPI> : (const void*)gemv_kernel<M, G, WPI>;
    const size_t smem = (size_t)M * K * sizeof(bf16) + (size_t)GEMV_WARPS * 2 * G * M * sizeof(float);
    static bool attr_done = false;   // per instantiation
    if (!attr_done) {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024) != cudaSuccess)
            return check_launch("tl_gemv_bf16 (smem attr)");
        attr_done = true;
    }
    TL_REQUIRE(smem <= 200 * 1024, TL_ERR_INVALID, "tl_gemv_bf16: M*K too large for shared memory (%zu B)", smem);
    const int n_items = ((N >> 1) + G - 1) / G;
    const int per_sm = smem > 100 * 1024 ? 1 : (smem > 64 * 1024 ? 2 : 4);
    int grid = (n_items + SLOTS - 1) / SLOTS;
    const int cap = sm_count() * per_sm;
    if (grid > cap) grid = cap;
    if constexpr (FP8)
        gemv_fp8_kernel<M, G, WPI><<<grid, GEMV_THREADS, smem, st>>>((const bf16*)x, (const fp8_e4m3*)W, (bf16*)y, N, K,
                                                                     (const bf16*)bias, (const bf16*)residual,
                                                                     (const bf16*)norm_w, eps, flags, scales);
    else
        gemv_kernel<M, G, WPI><<<grid, GEMV_THREADS, smem, st>>>((const bf16*)x, (const bf16*)W, (bf16*)y, N, K,
                                                                 (const bf16*)bias, (const bf16*)residual,
                                                                 (const bf16*)norm_w, eps, flags);
    return check_launch(FP8 ? "tl_gemv_fp8" : "tl_gemv_bf16");
}

template <typename WT, int M, int G>
static int dispatch_wpi(int wpi, const void* x, const void* W, const float* sc, void* y, int N, int K, const void* bias,
                        const void* residual, const void* norm_w, float eps, int flags, cudaStream_t st) {
    switch (wpi) {
        case 1: return launch_gemv<WT, M, G, 1>(x, W, sc, y, N, K, bias, residual, norm_w, eps, flags, st);
        case 2: return launch_gemv<WT, M, G, 2>(x, W, sc, y, N, K, bias, residual, norm_w, eps, flags, st);
        case 4: return launch_gemv<WT, M, G, 4>(x, W, sc, y, N, K, bias, residual, norm_w, eps, flags, st);
        default: return launch_gemv<WT, M, G, 8>(x, W, sc, y, N, K, bias, residual, norm_w, eps, flags, st);
    }
}

template <typename WT, int M>
static int dispatch_g(int g, int wpi, const void* x, const void* W, const float* sc, void* y, int N, int K,
                      const void* bias, const void* residual, const void* norm_w, float eps, int flags, cudaStream_t st) {
    switch (g) {
        case 4: return dispatch_wpi<WT, M, 4>(wpi, x, W, sc, y, N, K, bias, residual, norm_w, eps, flags, st);
        case 2: return dispatch_wpi<WT, M, 2>(wpi, x, W, sc, y, N, K, bias, residual, norm_w, eps, flags, st);
        default: return dispatch_wpi<WT, M, 1>(wpi, x, W, sc, y, N, K, bias, residual, norm_w, eps, flags, st);
    }
}

int gemv_stream_dispatch(const void* x, const void* W, void* y, int M, int N, int K, const void* bias,
                         const void* residual, const void* norm_w, float eps, int flags, unsigned* ctr, const void* pf_ptr,
                         size_t pf_bytes, cudaStream_t st);
int gemv_mma_dispatch(const void* x, const void* W, void* y, int M, int N, int K, const void* bias, const void* residual,
                      const void* norm_w, float eps, int flags, cudaStream_t st);
int gemv_stream_fp8_dispatch(const void* x, const void* W, const float* scales, void* y, int M, int N, int K,
                             const void* bias, const void* residual, const void* norm_w, float eps, int flags, unsigned* ctr,
                             const void* pf_ptr, size_t pf_bytes, cudaStream_t st);

static bool use_stream_kernel() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("TL_GEMV_IMPL");
        v = (e && e[0] == 'r') ? 0 : 1;     // TL_GEMV_IMPL=reg forces the register-streaming kernel (A/B tests)
    }
    return v == 1;
}

}  // namespace tl

namespace tl {

// Counter blocks for calls that bring none, taken round robin per device.  A block may be handed out again once no
// launch that used it can still run.  Launches on a stream overlap only through programmatic dependent launch: a launch
// starts once every CTA of the launch before it is running, and no CTA of it finishes before that launch has completed
// (the kernels launched this way wait for their predecessor: griddepcontrol.wait).  So the GEMV launches in flight at
// one time are all resident at once, each with at least one CTA of 288 threads: at most 7 per SM (2048 threads).  One
// call runs at most 2 launches, on different words of its block.  8 blocks per SM therefore never hand out a block that
// an earlier call may still be using.  The first call on a device allocates the pool, so it must not be captured.
constexpr int GEMV_MAX_DEVICES = 64;
static unsigned* g_ctr_pool[GEMV_MAX_DEVICES];
static int g_ctr_blocks[GEMV_MAX_DEVICES];
static std::atomic<unsigned> g_ctr_next[GEMV_MAX_DEVICES];
static std::mutex g_ctr_mu;

static unsigned* pool_counter() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= GEMV_MAX_DEVICES) return nullptr;
    if (!g_ctr_pool[dev]) {
        std::lock_guard<std::mutex> lk(g_ctr_mu);
        if (!g_ctr_pool[dev]) {
            const int n = 8 * sm_count();
            unsigned* p = nullptr;
            const size_t bytes = (size_t)n * TL_GEMV_COUNTER_WORDS * sizeof(unsigned);
            if (cudaMalloc(&p, bytes) != cudaSuccess) return nullptr;
            if (cudaMemset(p, 0, bytes) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) return nullptr;
            g_ctr_blocks[dev] = n;
            g_ctr_pool[dev] = p;
        }
    }
    const unsigned i = g_ctr_next[dev].fetch_add(1u) % (unsigned)g_ctr_blocks[dev];
    return g_ctr_pool[dev] + (size_t)i * TL_GEMV_COUNTER_WORDS;
}

// The passes of one decode Linear call (at most 4 rows each): the weight-streaming kernel, or the register-streaming
// kernel where x leaves its ring too few stages.  bf16 and FP8 weights take the same kernels, G and WPI on one shape.
template <typename WT>
static int gemv_passes(const void* x, const void* W, const float* scales, void* y, int M, int N, int K, const void* bias,
                       const void* residual, const void* norm_w, float eps, int flags, unsigned* counter,
                       const void* next_W, size_t next_bytes, cudaStream_t st) {
    const int nvec = K >> 3;
    int wpi = 1;
    while (wpi < 8 && (nvec + 32 * wpi - 1) / (32 * wpi) > 4) wpi <<= 1;
    const int slots = GEMV_WARPS / wpi;
    const int npairs = N >> 1;
    // larger G = more loads in flight per lane; shrink it until there are >= 4 rounds of items per CTA wave
    int g = 4;
    const int wave = sm_count() * 2 * slots;
    while (g > 1 && (npairs / g) < 4 * wave) g >>= 1;
    const int iters = (nvec + 32 * wpi - 1) / (32 * wpi);
    if (iters <= 4 && g < 2 && npairs >= 2 * wave) g = 2;
    // the M template is rounded up to 1/2/4/8 and the surplus rows are never written because the epilogue
    // indexes only m < M... (rows beyond M would read x out of bounds), so dispatch exactly for 1..4 and
    // split larger M into two calls.
    // the launches of one call may overlap under programmatic dependent launch: each takes its own two counter words
    auto run = [&](int m, const bf16* xx, bf16* yy, const bf16* rr, unsigned* ctr, bool last) -> int {
        if (use_stream_kernel()) {
            const void* pf = last ? next_W : nullptr;
            const size_t pfb = last && next_W ? next_bytes : 0;
            const int rc = sizeof(WT) == 1
                ? gemv_stream_fp8_dispatch(xx, W, scales, yy, m, N, K, bias, rr, norm_w, eps, flags, ctr, pf, pfb, st)
                : gemv_stream_dispatch(xx, W, yy, m, N, K, bias, rr, norm_w, eps, flags, ctr, pf, pfb, st);
            if (rc != 1) return rc;
        }
        switch (m) {
            case 1: return dispatch_g<WT, 1>(g, wpi, xx, W, scales, yy, N, K, bias, rr, norm_w, eps, flags, st);
            case 2: return dispatch_g<WT, 2>(g, wpi, xx, W, scales, yy, N, K, bias, rr, norm_w, eps, flags, st);
            case 3: return dispatch_g<WT, 3>(g, wpi, xx, W, scales, yy, N, K, bias, rr, norm_w, eps, flags, st);
            default: return dispatch_g<WT, 4>(g, wpi, xx, W, scales, yy, N, K, bias, rr, norm_w, eps, flags, st);
        }
    };
    const int n_out = (flags & TL_EPI_SWIGLU) ? N / 2 : N;
    int done = 0;
    while (done < M) {
        const int m = (M - done) > 4 ? 4 : (M - done);
        int rc = run(m, (const bf16*)x + (size_t)done * K, (bf16*)y + (size_t)done * n_out,
                     residual ? (const bf16*)residual + (size_t)done * N : nullptr, counter + 2 * (done / 4), done + m == M);
        if (rc != TL_OK) return rc;
        done += m;
    }
    return TL_OK;
}

}  // namespace tl

extern "C" int tl_gemv_bf16_pf(const void* x, const void* W, void* y, int M, int N, int K, const void* bias,
                               const void* residual, const void* norm_w, float eps, int flags, const void* next_W,
                               size_t next_bytes, void* stream) {
    return tl_gemv_bf16_ctr(x, W, y, M, N, K, bias, residual, norm_w, eps, flags, nullptr, next_W, next_bytes, stream);
}

extern "C" int tl_gemv_bf16(const void* x, const void* W, void* y, int M, int N, int K, const void* bias,
                            const void* residual, const void* norm_w, float eps, int flags, void* stream) {
    return tl_gemv_bf16_ctr(x, W, y, M, N, K, bias, residual, norm_w, eps, flags, nullptr, nullptr, 0, stream);
}

extern "C" int tl_gemv_bf16_ctr(const void* x, const void* W, void* y, int M, int N, int K, const void* bias,
                                const void* residual, const void* norm_w, float eps, int flags, unsigned* counter,
                                const void* next_W, size_t next_bytes, void* stream) {
    using namespace tl;
    TL_REQUIRE(M >= 1 && M <= 8, TL_ERR_INVALID, "tl_gemv_bf16: M=%d outside 1..8 (use tl_gemm_bf16)", M);
    TL_REQUIRE(((uintptr_t)counter & 3) == 0, TL_ERR_INVALID, "tl_gemv_bf16: counter block not 4-byte aligned");
    TL_REQUIRE(K % 8 == 0 && N % 2 == 0 && N > 0 && K > 0, TL_ERR_INVALID,
               "tl_gemv_bf16: need K %% 8 == 0 and N even (N=%d K=%d)", N, K);
    TL_REQUIRE(!(flags & ~(TL_EPI_BIAS | TL_EPI_RESIDUAL | TL_EPI_SWIGLU)), TL_ERR_INVALID,
               "tl_gemv_bf16: unsupported flags 0x%x", flags);
    TL_REQUIRE(!((flags & TL_EPI_SWIGLU) && (flags & TL_EPI_RESIDUAL)), TL_ERR_INVALID,
               "tl_gemv_bf16: SWIGLU and RESIDUAL are exclusive");
    TL_REQUIRE(!(flags & TL_EPI_BIAS) || bias, TL_ERR_INVALID, "tl_gemv_bf16: BIAS flag without bias pointer");
    TL_REQUIRE(!(flags & TL_EPI_RESIDUAL) || residual, TL_ERR_INVALID, "tl_gemv_bf16: RESIDUAL flag without pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (!counter && use_stream_kernel()) {
        counter = pool_counter();
        if (!counter) cudaGetLastError();
        TL_REQUIRE(counter, TL_ERR_CUDA, "tl_gemv_bf16: allocating the counter pool failed (first call on this device "
                   "inside a graph capture?)");
    }
    if (M >= 2 && use_stream_kernel()) {
        // 2..8 rows on mma.sync (gemv_mma.cu): opt-in; its per-row 1-2 KB bulk copies limit how fast an SM can issue
        // them, and it has not been compared with the CUDA-core stream kernel on H100.
        const char* e = getenv("TL_GEMV_MMA");
        if (e && e[0] == '1') {
            const int rc = gemv_mma_dispatch(x, W, y, M, N, K, bias, residual, norm_w, eps, flags, st);
            if (rc != 1) return rc;
        }
    }
    return tl::gemv_passes<bf16>(x, W, nullptr, y, M, N, K, bias, residual, norm_w, eps, flags, counter, next_W,
                                 next_bytes, st);
}

extern "C" int tl_gemv_fp8(const void* x, const void* W, const float* scales, void* y, int M, int N, int K, const void* bias,
                           const void* residual, const void* norm_w, float eps, int flags, void* stream) {
    return tl_gemv_fp8_ctr(x, W, scales, y, M, N, K, bias, residual, norm_w, eps, flags, nullptr, nullptr, 0, stream);
}

extern "C" int tl_gemv_fp8_ctr(const void* x, const void* W, const float* scales, void* y, int M, int N, int K,
                               const void* bias, const void* residual, const void* norm_w, float eps, int flags,
                               unsigned* counter, const void* next_W, size_t next_bytes, void* stream) {
    using namespace tl;
    TL_REQUIRE(M >= 1 && M <= 8, TL_ERR_INVALID, "tl_gemv_fp8: M=%d outside 1..8 (dequantize and use tl_gemm_bf16)", M);
    TL_REQUIRE(((uintptr_t)counter & 3) == 0, TL_ERR_INVALID, "tl_gemv_fp8: counter block not 4-byte aligned");
    TL_REQUIRE(K % TL_FP8_BLOCK == 0 && N % 2 == 0 && N > 0 && K > 0, TL_ERR_INVALID,
               "tl_gemv_fp8: need K %% %d == 0 and N even (N=%d K=%d)", TL_FP8_BLOCK, N, K);
    TL_REQUIRE(((uintptr_t)W & 15) == 0 && ((uintptr_t)scales & 3) == 0 && scales, TL_ERR_INVALID,
               "tl_gemv_fp8: W must be 16-byte aligned and scales non-NULL and 4-byte aligned");
    TL_REQUIRE(!(flags & ~(TL_EPI_BIAS | TL_EPI_RESIDUAL | TL_EPI_SWIGLU)), TL_ERR_INVALID,
               "tl_gemv_fp8: unsupported flags 0x%x", flags);
    TL_REQUIRE(!((flags & TL_EPI_SWIGLU) && (flags & TL_EPI_RESIDUAL)), TL_ERR_INVALID,
               "tl_gemv_fp8: SWIGLU and RESIDUAL are exclusive");
    TL_REQUIRE(!(flags & TL_EPI_BIAS) || bias, TL_ERR_INVALID, "tl_gemv_fp8: BIAS flag without bias pointer");
    TL_REQUIRE(!(flags & TL_EPI_RESIDUAL) || residual, TL_ERR_INVALID, "tl_gemv_fp8: RESIDUAL flag without pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (!counter) {
        counter = pool_counter();
        if (!counter) cudaGetLastError();
        TL_REQUIRE(counter, TL_ERR_CUDA, "tl_gemv_fp8: allocating the counter pool failed (first call on this device "
                   "inside a graph capture?)");
    }
    return gemv_passes<fp8_e4m3>(x, W, scales, y, M, N, K, bias, residual, norm_w, eps, flags, counter, next_W,
                                 next_bytes, st);
}
