// nn.Linear and its gradients as one persistent, warp-specialised wgmma GEMM (sm_90a).
//
//   C[M,N] (+)= A[M,K] · B[N,K]^T        bf16 operands, fp32 accumulation in registers
//
// CTA = 3 warpgroups: warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 = consumers, each issuing
// m64nBNk16 wgmma for one 64-row half of the 128 x BN output tile and running its epilogue.  BLOCK_K = 64 (one 128-byte
// swizzle atom of bf16), STAGES-deep smem ring fed by cp.async.bulk.tensor; the producer runs ahead into the next tile
// while the consumers run the epilogue of the current one.  Operands may be K-major (row-major [rows, K]) or MN-major
// (row-major [K, rows], wgmma's transpose bits) so the same kernel serves forward (x·W^T), dgrad (dy·W) and
// wgrad (dy^T·x) without transposes.
// Tensor-core roofline: 2*M*N*K flops per launch.
#include <stdlib.h>

#include <mutex>
#include <unordered_map>

#include "gemm_common.cuh"

namespace tl {

constexpr int GEMM_THREADS = 384;

// ---------------------------------------------------------------------------------------- tensor maps (host)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
        else
            cudaGetLastError();
    });
    return fn;
}

struct MapKey {
    const void* ptr;
    uint64_t inner, outer, ld;
    uint32_t box_inner, box_outer;
    bool operator==(const MapKey& o) const {
        return ptr == o.ptr && inner == o.inner && outer == o.outer && ld == o.ld && box_inner == o.box_inner &&
               box_outer == o.box_outer;
    }
};
struct MapKeyHash {
    size_t operator()(const MapKey& k) const {
        size_t h = (size_t)k.ptr;
        h = h * 1000003u ^ k.inner;
        h = h * 1000003u ^ k.outer;
        h = h * 1000003u ^ k.ld;
        h = h * 1000003u ^ ((uint64_t)k.box_inner << 32 | k.box_outer);
        return h;
    }
};

// 2-D bf16 row-major tensor [outer, inner] with leading dimension ld (elements); 128B-swizzled boxes
int make_tensor_map(CUtensorMap* out, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_inner,
                    uint32_t box_outer) {
    static std::mutex mu;
    static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
    MapKey key{ptr, inner, outer, ld, box_inner, box_outer};
    {
        std::lock_guard<std::mutex> g(mu);
        auto it = cache.find(key);
        if (it != cache.end()) {
            *out = it->second;
            return TL_OK;
        }
    }
    EncodeTiledFn enc = get_encode_fn();
    TL_REQUIRE(enc != nullptr, TL_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
    TL_REQUIRE(((uintptr_t)ptr & 15) == 0 && (ld * 2) % 16 == 0, TL_ERR_INVALID,
               "GEMM operand must be 16-byte aligned with a 16-byte-multiple row pitch (ptr=%p ld=%llu)", ptr,
               (unsigned long long)ld);
    cuuint64_t dims[2] = {inner, outer};
    cuuint64_t strides[1] = {ld * 2};
    cuuint32_t box[2] = {box_inner, box_outer};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    TL_REQUIRE(r == CUDA_SUCCESS, TL_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) inner=%llu outer=%llu ld=%llu",
               (int)r, (unsigned long long)inner, (unsigned long long)outer, (unsigned long long)ld);
    std::lock_guard<std::mutex> g(mu);
    if (cache.size() > 4096) cache.clear();
    cache[key] = *out;
    return TL_OK;
}

// ---------------------------------------------------------------------------------------- kernel
// Accumulators of one consumer warpgroup (64 x BN fp32) are written to a padded fp32 tile in shared memory and read back
// one row per lane for the shared epilogue; after that read the same bytes serve as the per-warp store staging tiles.
template <int BN>
struct GemmCfg {
    static constexpr int A_BYTES = BM * BK * 2;         // 16 KB
    static constexpr int B_BYTES = BN * BK * 2;         // 4 / 16 KB
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int STAGES = (BN == 128) ? 4 : 8;
    static constexpr int ACC_PITCH = BN + 4;            // floats; row-per-lane float4 reads are conflict-free
    static constexpr int ACC_BYTES = 64 * ACC_PITCH * 4;   // per consumer warpgroup
    static constexpr int UNITS = BN >= 64 ? 2 * (BN / 64) : 2;   // (row half, 64-column chunk) epilogue units per warpgroup
    static_assert(UNITS <= 4 && UNITS * EPI_STAGE_BYTES <= ACC_BYTES, "epilogue staging must fit in the accumulator tile");
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 2 * ACC_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
};

__device__ __forceinline__ void named_bar_sync(int id, int threads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

template <int BN, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, void* __restrict__ Cv,
                 int M, int N, int K, int ldc, const bf16* __restrict__ bias, const bf16* __restrict__ residual,
                 int ldr, int flags, int k_splits, int kb_per) {
    using Cfg = GemmCfg<BN>;
    extern __shared__ unsigned char smem_dyn[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    float* acc_tile = reinterpret_cast<float*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES);   // [2][64][ACC_PITCH]
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES + 2 * Cfg::ACC_BYTES);
    uint64_t* full_bar = bars;                         // [STAGES]
    uint64_t* empty_bar = bars + Cfg::STAGES;          // [STAGES]

    const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles_m = (M + BM - 1) / BM, tiles_n = (N + BN - 1) / BN;
    // split-K (weight-streaming regime, few output tiles): work item = (tile, k range); partial sums go to an fp32
    // workspace Cv[split][M][N] and a small reduce kernel applies the epilogue
    const int mn_tiles = tiles_m * tiles_n;
    const int total_tiles = mn_tiles * k_splits;
    const int num_k = (K + BK - 1) / BK;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < Cfg::STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 8);     // one arrive per consumer warp
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        // ===================================================================== TMA producer (one thread)
        if (threadIdx.x == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
                const int ks = t / mn_tiles, tt = t - ks * mn_tiles;
                const int m0 = (tt % tiles_m) * BM, n0 = (tt / tiles_m) * BN;
                const int kb0 = ks * kb_per, kb1 = min(num_k, kb0 + kb_per);
                for (int kb = kb0; kb < kb1; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    unsigned char* sa = smem + stage * Cfg::STAGE_BYTES;
                    unsigned char* sb = sa + Cfg::A_BYTES;
                    mbar_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
                    if (!A_MN) {
                        tma_load_2d(sa, &tmA, &full_bar[stage], kb * BK, m0);
                    } else {
#pragma unroll
                        for (int j = 0; j < BM / 64; ++j)
                            tma_load_2d(sa + j * 8192, &tmA, &full_bar[stage], m0 + 64 * j, kb * BK);
                    }
                    if (!B_MN) {
                        tma_load_2d(sb, &tmB, &full_bar[stage], kb * BK, n0);
                    } else {
#pragma unroll
                        for (int j = 0; j < BN / 64; ++j)
                            tma_load_2d(sb + j * 8192, &tmB, &full_bar[stage], n0 + 64 * j, kb * BK);
                    }
                    if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    // ========================================================================= consumers: warpgroup 1 = rows 0..63,
    // warpgroup 2 = rows 64..127 of the 128 x BN tile; each issues m64nBNk16 wgmma on the shared ring
    const int cw = wg - 1;                     // consumer warpgroup
    const int wq = warp & 3;                   // warp within it
    float* my_acc = acc_tile + cw * 64 * Cfg::ACC_PITCH;
    int stage = 0;
    uint32_t phase = 0;
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        const int ks = t / mn_tiles, tt = t - ks * mn_tiles;
        const int m0 = (tt % tiles_m) * BM, n0 = (tt / tiles_m) * BN;
        const int kb0 = ks * kb_per, kb1 = min(num_k, kb0 + kb_per);
        const bool active = m0 + 64 * cw < M;  // warpgroup-uniform; rows beyond M are TMA zero-fill, not stored
        float d[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
        int prev = -1;
        for (int kb = kb0; kb < kb1; ++kb) {
            mbar_wait(&full_bar[stage], phase);
            {
                const uint32_t sa = smem_u32(smem + stage * Cfg::STAGE_BYTES) + (uint32_t)(cw * 8192);
                const uint32_t sb = smem_u32(smem + stage * Cfg::STAGE_BYTES + Cfg::A_BYTES);
                // K-major: 8-row groups 1024 B apart (SBO), LBO unused, k-step = 32 B inside the swizzle atom
                // MN-major: 64-element MN chunks 8192 B apart (LBO), 8-k groups 1024 B apart (SBO), k-step = 2 KB
                const uint64_t da = A_MN ? make_wgmma_desc_sw128(sa, 8192, 1024) : make_wgmma_desc_sw128(sa, 16, 1024);
                const uint64_t db = B_MN ? make_wgmma_desc_sw128(sb, 8192, 1024) : make_wgmma_desc_sw128(sb, 16, 1024);
                wgmma_fence_acc(d);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / 16; ++k) {
                    const uint64_t ak = da + (uint64_t)((A_MN ? 2048 : 32) * k >> 4);
                    const uint64_t bk = db + (uint64_t)((B_MN ? 2048 : 32) * k >> 4);
                    const uint32_t acc = (kb > kb0 || k > 0) ? 1u : 0u;
                    if constexpr (BN == 128) wgmma_m64n128<A_MN ? 1 : 0, B_MN ? 1 : 0>(*reinterpret_cast<float(*)[64]>(d), ak, bk, acc);
                    else wgmma_m64n32<A_MN ? 1 : 0, B_MN ? 1 : 0>(*reinterpret_cast<float(*)[16]>(d), ak, bk, acc);
                }
                wgmma_commit();
                wgmma_fence_acc(d);
                wgmma_wait<1>();                   // the previous stage's MMAs have retired: hand its slot back
            }
            if (prev >= 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[prev]);
            }
            prev = stage;
            if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_acc(d);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
        if (!active) continue;                  // no rows of this warpgroup in this tile (warpgroup-uniform)

        // ---- epilogue: fragments -> fp32 tile -> one row per lane -> shared epilogue (bias / SwiGLU / residual / ...)
#pragma unroll
        for (int i = 0; i < BN / 2; i += 2) {
            const int r = 16 * wq + (lane >> 2) + 8 * ((i >> 1) & 1);
            const int c = 8 * (i >> 2) + 2 * (lane & 3);
            *reinterpret_cast<float2*>(my_acc + r * Cfg::ACC_PITCH + c) = make_float2(d[i], d[i + 1]);
        }
        named_bar_sync(1 + cw, 128);
        const int rh = wq & 1, ch = wq >> 1;   // this warp's epilogue unit: rows [32*rh, +32), columns [64*ch, +64)
        const bool has_unit = wq < Cfg::UNITS;
        uint32_t r0[32], r1[32];
        if (has_unit) {
            const float* row = my_acc + (32 * rh + lane) * Cfg::ACC_PITCH + 64 * ch;
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
                const float4 v = *reinterpret_cast<const float4*>(row + j);
                r0[j] = __float_as_uint(v.x); r0[j + 1] = __float_as_uint(v.y); r0[j + 2] = __float_as_uint(v.z); r0[j + 3] = __float_as_uint(v.w);
            }
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (BN >= 64) v = *reinterpret_cast<const float4*>(row + 32 + j);
                r1[j] = __float_as_uint(v.x); r1[j + 1] = __float_as_uint(v.y); r1[j + 2] = __float_as_uint(v.z); r1[j + 3] = __float_as_uint(v.w);
            }
        }
        named_bar_sync(1 + cw, 128);            // the fp32 tile is free: reuse it as the store staging tiles
        if (has_unit) {
            void* Ct = k_splits > 1 ? (void*)(reinterpret_cast<float*>(Cv) + (size_t)ks * M * N) : Cv;
            unsigned char* stg = reinterpret_cast<unsigned char*>(my_acc) + wq * EPI_STAGE_BYTES;
            gemm_epilogue_chunk64(r0, r1, stg, Ct, m0 + 64 * cw + 32 * rh, lane, n0 + 64 * ch, M, N, ldc, bias, residual, ldr,
                                  flags, BN >= 64 ? 64 : BN);
        }
        named_bar_sync(1 + cw, 128);            // staging reads done before the next tile's fragments land
    }
}

template <int BN, bool A_MN, bool B_MN>
static int launch_gemm(const void* A, const void* B, void* C, int M, int N, int K, int lda, int ldb, int ldc,
                       const void* bias, const void* residual, int flags, cudaStream_t st, int k_splits = 1, int kb_per = 0) {
    using Cfg = GemmCfg<BN>;
    CUtensorMap tmA, tmB;
    int rc;
    // K-major operand [rows, K]: inner = K, box = (64, rows-per-tile).  MN-major operand [K, rows]: inner = rows,
    // box = (64 rows, 64 k).
    rc = A_MN ? make_tensor_map(&tmA, A, (uint64_t)M, (uint64_t)K, (uint64_t)lda, 64, BK)
              : make_tensor_map(&tmA, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda, BK, BM);
    if (rc != TL_OK) return rc;
    rc = B_MN ? make_tensor_map(&tmB, B, (uint64_t)N, (uint64_t)K, (uint64_t)ldb, 64, BK)
              : make_tensor_map(&tmB, B, (uint64_t)K, (uint64_t)N, (uint64_t)ldb, BK, BN);
    if (rc != TL_OK) return rc;
    auto kern = gemm_bf16_kernel<BN, A_MN, B_MN>;
    static bool attr_done = false;
    if (!attr_done) {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES) != cudaSuccess)
            return check_launch("tl_gemm_bf16 (smem attr)");
        attr_done = true;
    }
    const int tiles = ((M + BM - 1) / BM) * ((N + BN - 1) / BN) * k_splits;
    const int grid = tiles < sm_count() ? tiles : sm_count();
    const int ldr = ldc;
    if (kb_per <= 0) kb_per = (K + BK - 1) / BK;
    kern<<<grid, GEMM_THREADS, Cfg::SMEM_BYTES, st>>>(tmA, tmB, C, M, N, K, ldc, (const bf16*)bias,
                                                      (const bf16*)residual, ldr, flags, k_splits, kb_per);
    return check_launch("tl_gemm_bf16");
}

template <int BN>
static int dispatch_major(bool a_mn, bool b_mn, const void* A, const void* B, void* C, int M, int N, int K, int lda,
                          int ldb, int ldc, const void* bias, const void* residual, int flags, cudaStream_t st) {
    if (!a_mn && !b_mn) return launch_gemm<BN, false, false>(A, B, C, M, N, K, lda, ldb, ldc, bias, residual, flags, st);
    if (!a_mn && b_mn) return launch_gemm<BN, false, true>(A, B, C, M, N, K, lda, ldb, ldc, bias, residual, flags, st);
    if (a_mn && !b_mn) return launch_gemm<BN, true, false>(A, B, C, M, N, K, lda, ldb, ldc, bias, residual, flags, st);
    return launch_gemm<BN, true, true>(A, B, C, M, N, K, lda, ldb, ldc, bias, residual, flags, st);
}

// out = epilogue(sum_s ws[s][m][n]); one thread per 8 columns (4 outputs for SwiGLU)
__global__ void splitk_reduce_kernel(const float* __restrict__ ws, void* __restrict__ Cv, int M, int N, int ldc, int splits,
                                     const bf16* __restrict__ bias, const bf16* __restrict__ residual, int ldr, int flags) {
    const int groups = N >> 3;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)M * groups) return;
    const int m = (int)(idx / groups), c0 = (int)(idx - (long long)m * groups) * 8;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = 0.f;
    for (int s = 0; s < splits; ++s) {
        const float4* p = reinterpret_cast<const float4*>(ws + ((size_t)s * M + m) * N + c0);
        const float4 a = p[0], b = p[1];
        v[0] += a.x; v[1] += a.y; v[2] += a.z; v[3] += a.w; v[4] += b.x; v[5] += b.y; v[6] += b.z; v[7] += b.w;
    }
    if (flags & TL_EPI_BIAS) {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] += bf2f(bias[c0 + j]);
    }
    if (flags & TL_EPI_SWIGLU) {
        bf16* dst = reinterpret_cast<bf16*>(Cv) + (size_t)m * ldc + (c0 >> 1);
#pragma unroll
        for (int j = 0; j < 4; ++j) dst[j] = f2bf(rbf(silu_f(rbf(v[2 * j]))) * rbf(v[2 * j + 1]));
        return;
    }
    if (flags & TL_EPI_OUT_F32) {
        float* dst = reinterpret_cast<float*>(Cv) + (size_t)m * ldc + c0;
#pragma unroll
        for (int j = 0; j < 8; ++j) dst[j] = v[j] + ((flags & TL_EPI_ACCUM) ? dst[j] : 0.f);
        return;
    }
    bf16* dst = reinterpret_cast<bf16*>(Cv) + (size_t)m * ldc + c0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        float t = rbf(v[j]);
        if (flags & TL_EPI_RESIDUAL) t += bf2f(residual[(size_t)m * ldr + c0 + j]);
        if (flags & TL_EPI_ACCUM) t += bf2f(dst[j]);
        v[j] = t;
    }
    *reinterpret_cast<uint4*>(dst) = make_uint4(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]), pack_bf16(v[4], v[5]), pack_bf16(v[6], v[7]));
}

// split-K reduce + epilogue (bias / residual, bf16 out) + the RMSNorm that follows the Linear, one CTA per row:
// C[m,:] = bf16(bf16(sum_s ws[s][m][:] + bias) + residual[m,:]);  Hn[m,:] = norm_w * bf16(C[m,:] * rstd(C[m,:])).
// 512 threads per row: one CTA serves a whole row (the norm needs all of it) and only M <= 128 CTAs exist, so the pass is
// latency-bound; every thread issues all of its 16 partial loads at once.  The sum of squares is
// reduced in a different order than rmsnorm_fwd_kernel's, i.e. Hn may differ from the unfused path in a last bf16 bit.
constexpr int RN_THREADS = 512;
constexpr int RN_MAXV = 2;
__global__ void __launch_bounds__(RN_THREADS)
splitk_reduce_norm_kernel(const float* __restrict__ ws, bf16* __restrict__ C, int M, int N, int ldc, int splits,
                          const bf16* __restrict__ bias, const bf16* __restrict__ residual, int ldr, int flags,
                          const bf16* __restrict__ norm_w, float eps, bf16* __restrict__ Hn) {
    const int m = blockIdx.x;
    const int nvec = N >> 3;
    uint4 xv[RN_MAXV];
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < RN_MAXV; ++i) {
        const int idx = threadIdx.x + i * RN_THREADS;
        if (idx < nvec) {
            const int c0 = idx * 8;
            float v[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = 0.f;
            // all partial loads of this column group are issued before the first add (one CTA serves a whole row, so
            // memory-level parallelism per thread is what keeps this pass short); summed in split order like the
            // stand-alone reduce kernel
            float4 pa[8], pb[8];
#pragma unroll
            for (int s = 0; s < 8; ++s) {
                if (s < splits) {
                    const float4* p = reinterpret_cast<const float4*>(ws + ((size_t)s * M + m) * N + c0);
                    pa[s] = __ldcs(p);
                    pb[s] = __ldcs(p + 1);
                }
            }
#pragma unroll
            for (int s = 0; s < 8; ++s) {
                if (s < splits) {
                    v[0] += pa[s].x; v[1] += pa[s].y; v[2] += pa[s].z; v[3] += pa[s].w;
                    v[4] += pb[s].x; v[5] += pb[s].y; v[6] += pb[s].z; v[7] += pb[s].w;
                }
            }
            if (flags & TL_EPI_BIAS) {
                const uint4 bb = *reinterpret_cast<const uint4*>(bias + c0);
                const uint32_t* b32 = reinterpret_cast<const uint32_t*>(&bb);
#pragma unroll
                for (int j = 0; j < 4; ++j) { v[2 * j] += bf16_lo(b32[j]); v[2 * j + 1] += bf16_hi(b32[j]); }
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = rbf(v[j]);
            if (flags & TL_EPI_RESIDUAL) {
                const uint4 rr = *reinterpret_cast<const uint4*>(residual + (size_t)m * ldr + c0);
                const uint32_t* r32 = reinterpret_cast<const uint32_t*>(&rr);
#pragma unroll
                for (int j = 0; j < 4; ++j) { v[2 * j] += bf16_lo(r32[j]); v[2 * j + 1] += bf16_hi(r32[j]); }
            }
            xv[i] = make_uint4(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]), pack_bf16(v[4], v[5]), pack_bf16(v[6], v[7]));
            *reinterpret_cast<uint4*>(C + (size_t)m * ldc + c0) = xv[i];
            const uint32_t* u = reinterpret_cast<const uint32_t*>(&xv[i]);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float a = bf16_lo(u[j]), b = bf16_hi(u[j]);
                ss += a * a + b * b;
            }
        }
    }
    __shared__ float red[RN_THREADS / 32];
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int i = 0; i < RN_THREADS / 32; ++i) tot += red[i];
    const float rstd = 1.0f / sqrtf(tot / (float)N + eps);
#pragma unroll
    for (int i = 0; i < RN_MAXV; ++i) {
        const int idx = threadIdx.x + i * RN_THREADS;
        if (idx < nvec) {
            const uint4 wv = reinterpret_cast<const uint4*>(norm_w)[idx];
            uint4 o;
            const uint32_t* u = reinterpret_cast<const uint32_t*>(&xv[i]);
            const uint32_t* g = reinterpret_cast<const uint32_t*>(&wv);
            uint32_t* ou = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float a = rbf(bf16_lo(u[j]) * rstd), b = rbf(bf16_hi(u[j]) * rstd);
                ou[j] = pack_bf16(bf16_lo(g[j]) * a, bf16_hi(g[j]) * b);
            }
            reinterpret_cast<uint4*>(Hn + (size_t)m * N)[idx] = o;
        }
    }
}

// The argument checks of tl_gemm_bf16, made by tl_gemm_bf16_ws_norm too before it chooses the split-K path, which
// would otherwise accept (and silently mis-execute) a combination tl_gemm_bf16 rejects.
static int check_gemm_args(int M, int N, int K, int lda, int ldb, int ldc, const void* bias, const void* residual, int flags) {
    TL_REQUIRE(M > 0 && N > 0 && K > 0, TL_ERR_INVALID, "tl_gemm_bf16: empty problem M=%d N=%d K=%d", M, N, K);
    TL_REQUIRE(N % 8 == 0, TL_ERR_INVALID, "tl_gemm_bf16: N must be a multiple of 8 (N=%d)", N);
    TL_REQUIRE(K % 8 == 0 || ((flags & TL_A_MN_MAJOR) && (flags & TL_B_MN_MAJOR)), TL_ERR_INVALID,
               "tl_gemm_bf16: K must be a multiple of 8 for K-major operands (K=%d)", K);
    TL_REQUIRE(!(flags & TL_EPI_BIAS) || bias, TL_ERR_INVALID, "tl_gemm_bf16: BIAS flag without bias pointer");
    TL_REQUIRE(!(flags & TL_EPI_RESIDUAL) || residual, TL_ERR_INVALID, "tl_gemm_bf16: RESIDUAL flag without pointer");
    const bool swiglu = flags & TL_EPI_SWIGLU;
    TL_REQUIRE(!swiglu || !(flags & (TL_EPI_RESIDUAL | TL_EPI_OUT_F32 | TL_EPI_ACCUM)), TL_ERR_INVALID,
               "tl_gemm_bf16: SWIGLU excludes RESIDUAL/OUT_F32/ACCUM");
    TL_REQUIRE(!swiglu || N % 16 == 0, TL_ERR_INVALID, "tl_gemm_bf16: SWIGLU needs N %% 16 == 0");
    const int c_cols = swiglu ? N / 2 : N;
    TL_REQUIRE(ldc >= c_cols && ldc % 8 == 0, TL_ERR_INVALID, "tl_gemm_bf16: ldc=%d too small / unaligned", ldc);
    const bool a_mn = flags & TL_A_MN_MAJOR, b_mn = flags & TL_B_MN_MAJOR;
    TL_REQUIRE(lda >= (a_mn ? M : K) && ldb >= (b_mn ? N : K), TL_ERR_INVALID, "tl_gemm_bf16: lda/ldb too small");
    TL_REQUIRE((!a_mn || M % 8 == 0), TL_ERR_INVALID, "tl_gemm_bf16: MN-major A needs M %% 8 == 0");
    return TL_OK;
}

}  // namespace tl

extern "C" size_t tl_gemm_splitk_ws(int M, int N) { return (size_t)8 * (size_t)(M > 128 ? 0 : M) * (size_t)N * sizeof(float); }

extern "C" int tl_gemm_bf16(const void* A, const void* B, void* C, int M, int N, int K, int lda, int ldb, int ldc,
                            const void* bias, const void* residual, int flags, void* stream);

// Same as tl_gemm_bf16; with a workspace the weight-streaming regime (M <= 128, K-major operands, too few output tiles to
// occupy every SM) is split along K so that all SMs stream weights, then reduced with the epilogue applied once.
extern "C" int tl_gemm_bf16_ws_norm(const void* A, const void* B, void* C, int M, int N, int K, int lda, int ldb, int ldc,
                                    const void* bias, const void* residual, int flags, void* workspace, size_t ws_bytes,
                                    const void* norm_w, float eps, void* H_out, void* stream);
extern "C" int tl_rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd_out, int rows, int H, float eps, void* stream);

extern "C" int tl_gemm_bf16_ws(const void* A, const void* B, void* C, int M, int N, int K, int lda, int ldb, int ldc,
                               const void* bias, const void* residual, int flags, void* workspace, size_t ws_bytes, void* stream) {
    return tl_gemm_bf16_ws_norm(A, B, C, M, N, K, lda, ldb, ldc, bias, residual, flags, workspace, ws_bytes, nullptr, 0.f, nullptr,
                                stream);
}

// ... and, when norm_w != NULL, H_out[M,N] = RMSNorm(C) * norm_w (the norm that follows this Linear in the decoder layer,
// N <= 8192): fused into the split-K reduce pass when that path is taken, a separate tl_rmsnorm_fwd launch otherwise.
extern "C" int tl_gemm_bf16_ws_norm(const void* A, const void* B, void* C, int M, int N, int K, int lda, int ldb, int ldc,
                                    const void* bias, const void* residual, int flags, void* workspace, size_t ws_bytes,
                                    const void* norm_w, float eps, void* H_out, void* stream) {
    using namespace tl;
    TL_REQUIRE(!norm_w || (H_out && ldc == N && !(flags & (TL_EPI_SWIGLU | TL_EPI_OUT_F32 | TL_EPI_ACCUM))), TL_ERR_INVALID,
               "tl_gemm_bf16_ws_norm: the fused norm needs H_out, ldc == N and a plain bf16 (bias/residual) epilogue");
    // both norm passes (the fused reduce and tl_rmsnorm_fwd) hold a whole row in registers: reject wider rows before
    // anything is launched, rather than after C has been written
    TL_REQUIRE(!norm_w || N <= RN_THREADS * RN_MAXV * 8, TL_ERR_INVALID, "tl_gemm_bf16_ws_norm: the fused norm needs N <= %d (N=%d)",
               RN_THREADS * RN_MAXV * 8, N);
    const int arg_rc = check_gemm_args(M, N, K, lda, ldb, ldc, bias, residual, flags);
    if (arg_rc != TL_OK) return arg_rc;
    const int tiles_n = (N + 127) / 128, num_k = (K + BK - 1) / BK;
    const bool plain = !(flags & (TL_A_MN_MAJOR | TL_B_MN_MAJOR));
    if (workspace && plain && M > 0 && M <= BM && K % 8 == 0 && N % 8 == 0 && tiles_n * 2 <= sm_count() && num_k >= 16) {
        int splits = sm_count() / tiles_n;
        if (splits > 8) splits = 8;
        int kb_per = (num_k + splits - 1) / splits;
        if (kb_per < 8) kb_per = 8;
        splits = (num_k + kb_per - 1) / kb_per;
        if (splits > 1 && ws_bytes >= (size_t)splits * M * N * sizeof(float)) {
            cudaStream_t st = (cudaStream_t)stream;
            int rc = launch_gemm<128, false, false>(A, B, workspace, M, N, K, lda, ldb, N, nullptr, nullptr, TL_EPI_OUT_F32, st,
                                                    splits, kb_per);
            if (rc != TL_OK) return rc;
            if (norm_w) {
                splitk_reduce_norm_kernel<<<M, RN_THREADS, 0, st>>>((const float*)workspace, (bf16*)C, M, N, ldc, splits,
                                                                    (const bf16*)bias, (const bf16*)residual, ldc, flags,
                                                                    (const bf16*)norm_w, eps, (bf16*)H_out);
                return check_launch("tl_gemm_bf16_ws_norm (reduce + norm)");
            }
            const long long items = (long long)M * (N >> 3);
            splitk_reduce_kernel<<<(unsigned)((items + 255) / 256), 256, 0, st>>>((const float*)workspace, C, M, N, ldc, splits,
                                                                                  (const bf16*)bias, (const bf16*)residual, ldc, flags);
            return check_launch("tl_gemm_bf16_ws (reduce)");
        }
    }
    int rc = tl_gemm_bf16(A, B, C, M, N, K, lda, ldb, ldc, bias, residual, flags, stream);
    if (rc != TL_OK || !norm_w) return rc;
    return tl_rmsnorm_fwd(C, norm_w, H_out, nullptr, M, N, eps, stream);
}

extern "C" int tl_gemm_bf16(const void* A, const void* B, void* C, int M, int N, int K, int lda, int ldb, int ldc,
                            const void* bias, const void* residual, int flags, void* stream) {
    using namespace tl;
    const int rc = check_gemm_args(M, N, K, lda, ldb, ldc, bias, residual, flags);
    if (rc != TL_OK) return rc;
    const bool a_mn = flags & TL_A_MN_MAJOR, b_mn = flags & TL_B_MN_MAJOR;
    cudaStream_t st = (cudaStream_t)stream;
    // few rows (M <= 128) and not enough 128-wide tiles to occupy every SM twice: 32-wide tiles (weight streaming)
    if (M <= BM && !b_mn && (long long)((N + 127) / 128) < 2LL * sm_count() && N % 32 == 0)
        return dispatch_major<32>(a_mn, b_mn, A, B, C, M, N, K, lda, ldb, ldc, bias, residual, flags, st);
    return dispatch_major<128>(a_mn, b_mn, A, B, C, M, N, K, lda, ldb, ldc, bias, residual, flags, st);
}
