// Decode-shaped Linear for 2..8 rows: the same persistent bulk-copy weight stream as gemv_stream.cu, but the dot
// products run on the tensor cores (mma.sync m16n8k16: 16 weight rows x 16 k  times  16 k x 8 batch rows), because at
// M >= 2 the fp32 FMA + bf16->fp32 conversion work of the CUDA-core kernel (not HBM) becomes the limit
// (and needs two passes at M = 8).
//
// Work unit = 16 consecutive weight rows (8 gate/up pairs).  A ring stage holds one K chunk of a unit: 16 row segments
// copied by cp.async.bulk into a padded pitch (conflict-free ldmatrix).  x (optionally RMS-normalised, HF rounding) is
// staged once per CTA as [8][K] bf16 (rows >= M are zero).  Stage -> warp mapping and barrier discipline are those of
// gemv_stream.cu (n_stages % NW == 0, every barrier has one waiting warp).
// Accumulation order differs from the CUDA-core kernel (k16 blocks inside the tensor core), so results agree with it to
// fp32 rounding, not bit for bit.
#include <stdlib.h>

#include "common.cuh"

namespace tl {

constexpr int GM_CONSUMER_WARPS = 8;
constexpr int GM_THREADS = (GM_CONSUMER_WARPS + 1) * 32;
constexpr int GM_KC = 1024;                      // K chunk (elements) per stage
constexpr int GM_PITCH = GM_KC * 2 + 16;         // bytes per staged weight row
constexpr int GM_STAGE_BYTES = 16 * GM_PITCH;    // 16,640 (weights only)
constexpr int GM_STAGE_BYTES_X = 24 * GM_PITCH;  // 24,960 (weights + the 8-row x chunk, for K too large to keep x resident)
constexpr int GM_MAX_STAGES = 16;

__device__ __forceinline__ void gm_ldsm4(uint32_t* r, const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void gm_mma(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(GM_THREADS, 1)
gemv_mma_kernel(const bf16* __restrict__ x, const bf16* __restrict__ W, bf16* __restrict__ y, int M, int N, int K,
                const bf16* __restrict__ bias, const bf16* __restrict__ residual, const bf16* __restrict__ norm_w, float eps,
                int flags, int n_stages, int NW, int xpitch, int x_in_stage) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int stage_bytes = x_in_stage ? GM_STAGE_BYTES_X : GM_STAGE_BYTES;
    unsigned char* ring = smem;                                                      // [n_stages][16 (+8)][GM_PITCH]
    unsigned char* xs = smem + (size_t)n_stages * stage_bytes;                       // [8][xpitch bytes] (resident-x mode)
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(xs + (x_in_stage ? 0 : (size_t)8 * xpitch));
    uint64_t* empty_bar = full_bar + GM_MAX_STAGES;
    __shared__ float s_part[GM_CONSUMER_WARPS][8];

    asm volatile("griddepcontrol.launch_dependents;");
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n_units_all = N >> 4;                                  // units of 16 rows
    const int u_begin = (int)((long long)blockIdx.x * n_units_all / gridDim.x);
    const int u_end = (int)((long long)(blockIdx.x + 1) * n_units_all / gridDim.x);
    const int n_units = u_end - u_begin;
    const int n_groups = (n_units + NW - 1) / NW;
    const int n_chunks = (K + GM_KC - 1) / GM_KC;

    if (tid == 0) {
        for (int s = 0; s < n_stages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 1);
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == GM_CONSUMER_WARPS) {
        // ================================================================= producer: lanes 0..15 copy one row segment each
        // (streamed-x mode also reads activations of the previous kernel: then the producer must wait for it as well)
        if (x_in_stage) asm volatile("griddepcontrol.wait;" ::: "memory");
        int stage = 0;
        uint32_t phase = 0;
        for (int g = 0; g < n_groups; ++g)
            for (int c = 0; c < n_chunks; ++c)
                for (int w = 0; w < NW; ++w) {
                    const int unit = g * NW + w;
                    const int k0 = c * GM_KC;
                    const uint32_t bytes = (uint32_t)min(GM_KC, K - k0) * 2u;
                    if (lane == 0) {
                        mbar_wait(&empty_bar[stage], phase ^ 1);
                        mbar_expect_tx(&full_bar[stage], unit < n_units ? (16u + (x_in_stage ? (uint32_t)M : 0u)) * bytes : 0u);
                    }
                    __syncwarp();
                    if (unit < n_units && lane < 16)
                        bulk_load_1d(ring + (size_t)stage * stage_bytes + (size_t)lane * GM_PITCH,
                                     W + ((size_t)(u_begin + unit) * 16 + lane) * K + k0, bytes, &full_bar[stage]);
                    if (unit < n_units && x_in_stage && lane >= 16 && lane < 16 + M)      // x rows ride along (L2-resident)
                        bulk_load_1d(ring + (size_t)stage * stage_bytes + (size_t)lane * GM_PITCH,
                                     x + (size_t)(lane - 16) * K + k0, bytes, &full_bar[stage]);
                    if (++stage == n_stages) { stage = 0; phase ^= 1; }
                }
        return;
    }

    // ===================================================================== consumers
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int nvec = K >> 3;
    if (!x_in_stage) {   // ---- stage x: [8][K] bf16 with row pitch xpitch; rows >= M are zero
        float rstd[8];
#pragma unroll
        for (int m = 0; m < 8; ++m) rstd[m] = 1.f;
        if (norm_w) {
            float ss[8];
#pragma unroll
            for (int m = 0; m < 8; ++m) ss[m] = 0.f;
            for (int v = tid; v < nvec; v += GM_CONSUMER_WARPS * 32) {
#pragma unroll
                for (int m = 0; m < 8; ++m) {
                    if (m < M) {
                        const uint4 u = reinterpret_cast<const uint4*>(x + (size_t)m * K)[v];
                        const uint32_t* u32 = reinterpret_cast<const uint32_t*>(&u);
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const float a = bf16_lo(u32[j]), b = bf16_hi(u32[j]);
                            ss[m] += a * a + b * b;
                        }
                    }
                }
            }
#pragma unroll
            for (int m = 0; m < 8; ++m) {
                const float t = warp_sum(ss[m]);
                if (lane == 0) s_part[warp][m] = t;
            }
            asm volatile("bar.sync 1, 256;" ::: "memory");
#pragma unroll
            for (int m = 0; m < 8; ++m) {
                float t = 0.f;
#pragma unroll
                for (int w = 0; w < GM_CONSUMER_WARPS; ++w) t += s_part[w][m];
                rstd[m] = 1.0f / sqrtf(t / (float)K + eps);
            }
        }
        for (int v = tid; v < nvec; v += GM_CONSUMER_WARPS * 32) {
            uint4 g = make_uint4(0, 0, 0, 0);
            if (norm_w) g = reinterpret_cast<const uint4*>(norm_w)[v];
            const uint32_t* g32 = reinterpret_cast<const uint32_t*>(&g);
#pragma unroll
            for (int m = 0; m < 8; ++m) {
                uint4 o = make_uint4(0, 0, 0, 0);
                if (m < M) {
                    const uint4 u = reinterpret_cast<const uint4*>(x + (size_t)m * K)[v];
                    if (norm_w) {
                        const uint32_t* u32 = reinterpret_cast<const uint32_t*>(&u);
                        uint32_t* o32 = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
                        for (int j = 0; j < 4; ++j)
                            o32[j] = pack_bf16(bf16_lo(g32[j]) * rbf(bf16_lo(u32[j]) * rstd[m]),
                                               bf16_hi(g32[j]) * rbf(bf16_hi(u32[j]) * rstd[m]));
                    } else {
                        o = u;
                    }
                }
                *reinterpret_cast<uint4*>(xs + (size_t)m * xpitch + (size_t)v * 16) = o;
            }
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
    }

    if (warp >= NW) return;
    const bool swiglu = flags & TL_EPI_SWIGLU;
    const int n_out = swiglu ? (N >> 1) : N;
    const int g8 = lane >> 2, t4 = lane & 3;
    int seq = warp;
    for (int g = 0; g < n_groups; ++g) {
        const int unit = g * NW + warp;
        const bool valid = unit < n_units;
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        for (int c = 0; c < n_chunks; ++c, seq += NW) {
            const int stage = seq % n_stages;
            const uint32_t phase = (uint32_t)(seq / n_stages) & 1u;
            mbar_wait(&full_bar[stage], phase);
            if (valid) {
                const unsigned char* wt = ring + (size_t)stage * stage_bytes;
                const int k0 = c * GM_KC;
                const int ksteps = (min(GM_KC, K - k0) + 15) >> 4;
#pragma unroll 4
                for (int ks = 0; ks < ksteps; ++ks) {
                    uint32_t a[4];
                    gm_ldsm4(a, wt + (size_t)(lane & 15) * GM_PITCH + (size_t)(ks * 16 + (lane >> 4) * 8) * 2);
                    const unsigned char* xb = x_in_stage ? wt + (size_t)(16 + g8) * GM_PITCH + (size_t)(ks * 16 + 2 * t4) * 2
                                                         : xs + (size_t)g8 * xpitch + (size_t)(k0 + ks * 16 + 2 * t4) * 2;
                    uint32_t b0 = 0u, b1 = 0u;
                    if (!x_in_stage || g8 < M) {            // rows >= M are not copied in streamed-x mode
                        b0 = *reinterpret_cast<const uint32_t*>(xb);
                        b1 = *reinterpret_cast<const uint32_t*>(xb + 16);
                    }
                    gm_mma(acc, a, b0, b1);
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[stage]);
        }
        if (!valid) continue;
        // ---- epilogue: acc[0..1] = (row g8, batch 2t4, 2t4+1), acc[2..3] = (row g8+8, same batches)
        const int row_base = (u_begin + unit) * 16;
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            const int row = row_base + g8 + hr * 8;
            float v0 = acc[2 * hr], v1 = acc[2 * hr + 1];
            if (flags & TL_EPI_BIAS) {
                const float bb = bf2f(bias[row]);
                v0 += bb;
                v1 += bb;
            }
            if (swiglu) {
                // pair (gate = even row, up = odd row): rows g8 and g8^1 live 4 lanes apart
                const float o0 = __shfl_xor_sync(0xffffffffu, v0, 4), o1 = __shfl_xor_sync(0xffffffffu, v1, 4);
                if ((g8 & 1) == 0) {
                    const int pair = row >> 1;
                    if (2 * t4 < M) y[(size_t)(2 * t4) * n_out + pair] = f2bf(rbf(silu_f(rbf(v0))) * rbf(o0));
                    if (2 * t4 + 1 < M) y[(size_t)(2 * t4 + 1) * n_out + pair] = f2bf(rbf(silu_f(rbf(v1))) * rbf(o1));
                }
            } else {
                float t0 = rbf(v0), t1 = rbf(v1);
                if (flags & TL_EPI_RESIDUAL) {
                    if (2 * t4 < M) t0 += bf2f(residual[(size_t)(2 * t4) * N + row]);
                    if (2 * t4 + 1 < M) t1 += bf2f(residual[(size_t)(2 * t4 + 1) * N + row]);
                }
                if (2 * t4 < M) y[(size_t)(2 * t4) * N + row] = f2bf(t0);
                if (2 * t4 + 1 < M) y[(size_t)(2 * t4 + 1) * N + row] = f2bf(t1);
            }
        }
    }
}

// returns TL_OK / error, or 1 = not applicable (caller falls back)
int gemv_mma_dispatch(const void* x, const void* W, void* y, int M, int N, int K, const void* bias, const void* residual,
                      const void* norm_w, float eps, int flags, cudaStream_t st) {
    if (M < 2 || M > 8 || N % 16 != 0 || K % 16 != 0 || ((uintptr_t)W & 15)) return 1;
    constexpr int SMEM_CAP = 220 * 1024;
    // x row pitch: K*2 bytes + 16 so that the 8 rows of a B fragment fall into different banks
    const int xpitch = K * 2 + 16;
    // resident x when it fits beside a useful ring, else (no norm prologue only) x chunks ride along in every stage
    int x_in_stage = 0;
    size_t fixed = (size_t)8 * xpitch + 2 * GM_MAX_STAGES * sizeof(uint64_t);
    if (fixed + 6 * (size_t)GM_STAGE_BYTES > (size_t)SMEM_CAP) {
        if (norm_w) return 1;
        x_in_stage = 1;
        fixed = 2 * GM_MAX_STAGES * sizeof(uint64_t);
    }
    const int stage_bytes = x_in_stage ? GM_STAGE_BYTES_X : GM_STAGE_BYTES;
    static bool attr_done = false;
    if (!attr_done) {
        if (cudaFuncSetAttribute(gemv_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_CAP) != cudaSuccess)
            return check_launch("tl_gemv_bf16/mma (smem attr)");
        attr_done = true;
    }
    int max_stages = (int)((SMEM_CAP - fixed) / stage_bytes);
    if (max_stages > GM_MAX_STAGES) max_stages = GM_MAX_STAGES;
    int n_stages = 0, NW = 0;
    for (int nw = GM_CONSUMER_WARPS; nw >= 4; --nw) {
        const int s = max_stages / nw * nw;
        if (s > n_stages) { n_stages = s; NW = nw; }
    }
    if (n_stages == 0) return 1;
    const size_t smem = (size_t)n_stages * stage_bytes + fixed;
    int grid = sm_count();
    if (grid > (N >> 4)) grid = N >> 4;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(GM_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    static int use_pdl = -1;
    if (use_pdl < 0) {
        const char* e = getenv("TL_PDL");
        use_pdl = (e && e[0] == '0') ? 0 : 1;
    }
    cfg.attrs = attr;
    cfg.numAttrs = use_pdl ? 1 : 0;
    cudaLaunchKernelEx(&cfg, gemv_mma_kernel, (const bf16*)x, (const bf16*)W, (bf16*)y, M, N, K, (const bf16*)bias,
                       (const bf16*)residual, (const bf16*)norm_w, eps, flags, n_stages, NW, xpitch, x_in_stage);
    return check_launch("tl_gemv_bf16/mma");
}

}  // namespace tl
