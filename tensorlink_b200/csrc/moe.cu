// Qwen3-MoE sparse MLP block (HF Qwen3MoeSparseMoeBlock, eager experts), sm_90a.
//
//   route     top-k of the fp32 softmax of each token's bf16 router logits; ids sorted ascending, fp32 weights
//             (optionally renormalised over the k picks).  For the grouped path also the plan: per-expert counts,
//             segment offsets padded to the GEMM's 128-row tile, the (token, slot) -> segment-row map and the
//             M-tile -> (expert, valid rows) table.  Tokens inside a segment are in ascending token order.
//   gather    h rows -> their segment rows (TMA cannot gather rows, so the grouped GEMM reads a packed A).
//   gemm      grouped wgmma GEMM: M-tile t of A multiplies expert tiles[t].x's weight slice (B rows e*N ..);
//             rows past the segment's valid count are never stored, empty tiles exit.  Same pipeline as
//             gemm_bf16_kernel (gemm.cu): one TMA producer warpgroup, two consumer warpgroups, the shared epilogue.
//   combine   out[t] = bf16(x[t] + acc), acc = +0, then for each pick in ascending expert order
//             acc = bf16(acc + bf16(fp32(y) * w)) — HF's bf16 zeros_like + index_add_ over the sorted expert_hit.
//   gemv      decode rows: stream only the picked experts' weights.  gate/up: one (row, pick) per grid row with the
//             SwiGLU epilogue; down: every output element computes its row's k products in ascending expert order
//             and applies the combine and the residual in its epilogue.
// Nothing is read back to the host: the decode and batched-decode steps stay graph-capturable.
#include <cuda.h>

#include "gemm_common.cuh"

namespace tl {

int make_tensor_map(CUtensorMap* out, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_inner,
                    uint32_t box_outer);

constexpr int MOE_MAX_E = 256;
constexpr int MOE_MAX_K = 16;
constexpr int MOE_PLAN_THREADS = 1024;

// ---------------------------------------------------------------------------------------- route: top-k per token
// One warp per token.  Selection compares the bf16 logits (softmax is monotonic; equal probabilities come from equal
// logits), ties toward the lower expert index.
__global__ void moe_topk_kernel(const bf16* __restrict__ logits, int32_t* __restrict__ ids, float* __restrict__ wts,
                                int N, int E, int k, int norm) {
    const int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (t >= N) return;
    constexpr int PER = MOE_MAX_E / 32;
    float l[PER];
    float m = -INFINITY;
#pragma unroll
    for (int j = 0; j < PER; ++j) {
        const int e = lane + 32 * j;
        l[j] = e < E ? bf2f(logits[(size_t)t * E + e]) : -INFINITY;
        m = fmaxf(m, l[j]);
    }
    m = warp_max(m);
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < PER; ++j)
        if (lane + 32 * j < E) s += expf(l[j] - m);
    s = warp_sum(s);
    int pick[MOE_MAX_K];
    float pv[MOE_MAX_K];
    for (int i = 0; i < k; ++i) {
        float bv = -INFINITY;
        int bi = 0x7fffffff;
#pragma unroll
        for (int j = 0; j < PER; ++j) {
            const int e = lane + 32 * j;
            if (e < E && (l[j] > bv || (l[j] == bv && e < bi))) { bv = l[j]; bi = e; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        pick[i] = bi;
        pv[i] = expf(bv - m) / s;
#pragma unroll
        for (int j = 0; j < PER; ++j)
            if (lane + 32 * j == bi) l[j] = -INFINITY;
    }
    if (lane != 0) return;
    float tot = 0.f;
    for (int i = 0; i < k; ++i) tot += pv[i];            // descending-probability order, as torch.topk returns them
    for (int i = 1; i < k; ++i) {                        // insertion sort by expert id
        const int pi = pick[i];
        const float pp = pv[i];
        int j = i - 1;
        while (j >= 0 && pick[j] > pi) { pick[j + 1] = pick[j]; pv[j + 1] = pv[j]; --j; }
        pick[j + 1] = pi;
        pv[j + 1] = pp;
    }
    for (int i = 0; i < k; ++i) {
        ids[(size_t)t * k + i] = pick[i];
        wts[(size_t)t * k + i] = norm ? pv[i] / tot : pv[i];
    }
}

// ---------------------------------------------------------------------------------------- route: grouped-GEMM plan
// One CTA.  Tokens go in chunks of 1024 (one per thread); a pick's place in its expert's segment = picks of that expert
// by earlier chunks + by earlier warps of this chunk + by earlier lanes of this warp.  Counts are sums, so the shared
// atomics do not make the order depend on timing.
__global__ void __launch_bounds__(MOE_PLAN_THREADS)
moe_plan_kernel(const int32_t* __restrict__ ids, int N, int E, int k, int32_t* __restrict__ counts,
                int32_t* __restrict__ offsets, int32_t* __restrict__ row_of, int32_t* __restrict__ tiles, int max_tiles) {
    __shared__ int wcnt[MOE_PLAN_THREADS / 32][MOE_MAX_E];
    __shared__ int tot[MOE_MAX_E];
    __shared__ int off[MOE_MAX_E + 1];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    for (int e = tid; e < E; e += blockDim.x) tot[e] = 0;
    for (int c0 = 0; c0 < N; c0 += MOE_PLAN_THREADS) {
        const int t = c0 + tid;
        int id[MOE_MAX_K], rank[MOE_MAX_K];
#pragma unroll
        for (int s = 0; s < MOE_MAX_K; ++s) {
            id[s] = (t < N && s < k) ? ids[(size_t)t * k + s] : -1;
            rank[s] = 0;
        }
        for (int i = tid; i < (MOE_PLAN_THREADS / 32) * MOE_MAX_E; i += blockDim.x) (&wcnt[0][0])[i] = 0;
        for (int l = 0; l < 31; ++l) {
#pragma unroll
            for (int s2 = 0; s2 < MOE_MAX_K; ++s2) {
                const int o = __shfl_sync(0xffffffffu, id[s2], l);
#pragma unroll
                for (int s = 0; s < MOE_MAX_K; ++s) rank[s] += (l < lane && o >= 0 && o == id[s]) ? 1 : 0;
            }
        }
        __syncthreads();
#pragma unroll
        for (int s = 0; s < MOE_MAX_K; ++s)
            if (id[s] >= 0) atomicAdd(&wcnt[warp][id[s]], 1);
        __syncthreads();
        for (int e = tid; e < E; e += blockDim.x) {
            int run = tot[e];
            for (int w = 0; w < MOE_PLAN_THREADS / 32; ++w) {
                const int c = wcnt[w][e];
                wcnt[w][e] = run;
                run += c;
            }
            tot[e] = run;
        }
        __syncthreads();
#pragma unroll
        for (int s = 0; s < MOE_MAX_K; ++s)
            if (id[s] >= 0) row_of[(size_t)t * k + s] = wcnt[warp][id[s]] + rank[s];   // segment-local for now
        __syncthreads();
    }
    if (tid == 0) {
        int o = 0;
        for (int e = 0; e < E; ++e) {
            off[e] = o;
            o += (tot[e] + BM - 1) / BM * BM;
        }
        off[E] = o;
    }
    __syncthreads();
    for (int e = tid; e < E; e += blockDim.x) counts[e] = tot[e];
    for (int e = tid; e <= E; e += blockDim.x) offsets[e] = off[e];
    for (long long i = tid; i < (long long)N * k; i += blockDim.x) row_of[i] += off[ids[i]];
    for (int tt = tid; tt < max_tiles; tt += blockDim.x) {
        const int r = tt * BM;
        int e = -1, valid = 0;
        if (r < off[E]) {
            int lo = 0, hi = E - 1;                      // last expert with off[e] <= r
            while (lo < hi) {
                const int mid = (lo + hi + 1) >> 1;
                if (off[mid] <= r) lo = mid; else hi = mid - 1;
            }
            e = lo;
            valid = min(BM, tot[e] - (r - off[e]));
        }
        tiles[2 * tt] = e;
        tiles[2 * tt + 1] = valid;
    }
}

// ---------------------------------------------------------------------------------------- gather / combine
__global__ void moe_gather_kernel(const bf16* __restrict__ h, const int32_t* __restrict__ row_of, bf16* __restrict__ hg,
                                  int k, int H) {
    const int i = blockIdx.x, t = i / k;
    const uint4* src = reinterpret_cast<const uint4*>(h + (size_t)t * H);
    uint4* dst = reinterpret_cast<uint4*>(hg + (size_t)row_of[i] * H);
    for (int c = threadIdx.x; c < H / 8; c += blockDim.x) dst[c] = src[c];
}

__device__ __forceinline__ float moe_add(float acc, float y, float w) { return rbf(acc + rbf(y * w)); }

__global__ void moe_combine_kernel(const bf16* __restrict__ y, const int32_t* __restrict__ row_of, const float* __restrict__ wts,
                                   const bf16* __restrict__ x, bf16* __restrict__ out, int k, int H) {
    const int t = blockIdx.x;
    for (int c = threadIdx.x * 2; c < H; c += blockDim.x * 2) {
        float a0 = 0.f, a1 = 0.f;
        for (int s = 0; s < k; ++s) {
            const float w = wts[(size_t)t * k + s];
            const uint32_t v = *reinterpret_cast<const uint32_t*>(y + (size_t)row_of[(size_t)t * k + s] * H + c);
            a0 = moe_add(a0, bf16_lo(v), w);
            a1 = moe_add(a1, bf16_hi(v), w);
        }
        const uint32_t xv = *reinterpret_cast<const uint32_t*>(x + (size_t)t * H + c);
        *reinterpret_cast<uint32_t*>(out + (size_t)t * H + c) = pack_bf16(bf16_lo(xv) + a0, bf16_hi(xv) + a1);
    }
}

// ---------------------------------------------------------------------------------------- grouped wgmma GEMM
constexpr int MG_THREADS = 384;
constexpr int MG_BN = 128;
constexpr int MG_STAGES = 4;
constexpr int MG_A_BYTES = BM * BK * 2;
constexpr int MG_STAGE_BYTES = MG_A_BYTES + MG_BN * BK * 2;
constexpr int MG_ACC_PITCH = MG_BN + 4;
constexpr int MG_ACC_BYTES = 64 * MG_ACC_PITCH * 4;
constexpr int MG_SMEM_BYTES = MG_STAGES * MG_STAGE_BYTES + 2 * MG_ACC_BYTES + 1024 + 256;

__device__ __forceinline__ void mg_bar_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

// C[r, :] = epilogue(A[r, :] · W[e]^T) for the valid rows r of every M-tile; W is [E*N, K], expert e's rows e*N..e*N+N-1.
__global__ void __launch_bounds__(MG_THREADS, 1)
moe_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, bf16* __restrict__ C,
                const int32_t* __restrict__ tiles, int max_tiles, int N, int K, int ldc, int flags) {
    extern __shared__ unsigned char smem_dyn[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    float* acc_tile = reinterpret_cast<float*>(smem + MG_STAGES * MG_STAGE_BYTES);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + MG_STAGES * MG_STAGE_BYTES + 2 * MG_ACC_BYTES);
    uint64_t* full_bar = bars;
    uint64_t* empty_bar = bars + MG_STAGES;
    const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles_n = N / MG_BN;
    const int total = max_tiles * tiles_n;
    const int num_k = (K + BK - 1) / BK;
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < MG_STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 8);
        }
        fence_barrier_init();
    }
    __syncthreads();
    if (wg == 0) {
        if (threadIdx.x == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int t = blockIdx.x; t < total; t += gridDim.x) {
                const int mt = t % max_tiles, e = tiles[2 * mt];
                if (e < 0) continue;
                const int m0 = mt * BM, b0 = e * N + (t / max_tiles) * MG_BN;
                for (int kb = 0; kb < num_k; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    unsigned char* sa = smem + stage * MG_STAGE_BYTES;
                    mbar_expect_tx(&full_bar[stage], MG_STAGE_BYTES);
                    tma_load_2d(sa, &tmA, &full_bar[stage], kb * BK, m0);
                    tma_load_2d(sa + MG_A_BYTES, &tmB, &full_bar[stage], kb * BK, b0);
                    if (++stage == MG_STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }
    const int cw = wg - 1, wq = warp & 3;
    float* my_acc = acc_tile + cw * 64 * MG_ACC_PITCH;
    int stage = 0;
    uint32_t phase = 0;
    for (int t = blockIdx.x; t < total; t += gridDim.x) {
        const int mt = t % max_tiles;
        if (tiles[2 * mt] < 0) continue;
        const int m0 = mt * BM, n0 = (t / max_tiles) * MG_BN;
        const int row_end = m0 + tiles[2 * mt + 1];
        const bool active = m0 + 64 * cw < row_end;
        float d[MG_BN / 2];
#pragma unroll
        for (int i = 0; i < MG_BN / 2; ++i) d[i] = 0.f;
        int prev = -1;
        for (int kb = 0; kb < num_k; ++kb) {
            mbar_wait(&full_bar[stage], phase);
            {
                const uint32_t sa = smem_u32(smem + stage * MG_STAGE_BYTES) + (uint32_t)(cw * 8192);
                const uint32_t sb = smem_u32(smem + stage * MG_STAGE_BYTES + MG_A_BYTES);
                const uint64_t da = make_wgmma_desc_sw128(sa, 16, 1024);
                const uint64_t db = make_wgmma_desc_sw128(sb, 16, 1024);
                wgmma_fence_acc(d);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / 16; ++k) {
                    const uint32_t acc = (kb > 0 || k > 0) ? 1u : 0u;
                    wgmma_m64n128<0, 0>(*reinterpret_cast<float(*)[64]>(d), da + (uint64_t)(32 * k >> 4),
                                        db + (uint64_t)(32 * k >> 4), acc);
                }
                wgmma_commit();
                wgmma_fence_acc(d);
                wgmma_wait<1>();
            }
            if (prev >= 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[prev]);
            }
            prev = stage;
            if (++stage == MG_STAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_acc(d);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
        if (!active) continue;
#pragma unroll
        for (int i = 0; i < MG_BN / 2; i += 2) {
            const int r = 16 * wq + (lane >> 2) + 8 * ((i >> 1) & 1);
            const int c = 8 * (i >> 2) + 2 * (lane & 3);
            *reinterpret_cast<float2*>(my_acc + r * MG_ACC_PITCH + c) = make_float2(d[i], d[i + 1]);
        }
        mg_bar_sync(1 + cw, 128);
        const int rh = wq & 1, ch = wq >> 1;
        uint32_t r0[32], r1[32];
        const float* row = my_acc + (32 * rh + lane) * MG_ACC_PITCH + 64 * ch;
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
            const float4 v = *reinterpret_cast<const float4*>(row + j);
            r0[j] = __float_as_uint(v.x); r0[j + 1] = __float_as_uint(v.y); r0[j + 2] = __float_as_uint(v.z); r0[j + 3] = __float_as_uint(v.w);
            const float4 u = *reinterpret_cast<const float4*>(row + 32 + j);
            r1[j] = __float_as_uint(u.x); r1[j + 1] = __float_as_uint(u.y); r1[j + 2] = __float_as_uint(u.z); r1[j + 3] = __float_as_uint(u.w);
        }
        mg_bar_sync(1 + cw, 128);
        unsigned char* stg = reinterpret_cast<unsigned char*>(my_acc) + wq * EPI_STAGE_BYTES;
        gemm_epilogue_chunk64(r0, r1, stg, C, m0 + 64 * cw + 32 * rh, lane, n0 + 64 * ch, row_end, N, ldc, nullptr, nullptr, 0,
                              flags, 64);
        mg_bar_sync(1 + cw, 128);
    }
}

// ---------------------------------------------------------------------------------------- expert GEMV (decode rows)
constexpr int MV_THREADS = 256;

// grid (ceil(I / 8), M*k): warp -> the (gate, up) row pair j of expert ids[r*k+s]; y[(r*k+s), j] = SwiGLU
__global__ void __launch_bounds__(MV_THREADS)
moe_gemv_gu_kernel(const bf16* __restrict__ x, const bf16* __restrict__ W, bf16* __restrict__ y, const int32_t* __restrict__ ids,
                   int k, int I, int K) {
    extern __shared__ uint4 xs[];
    const int rs = blockIdx.y, r = rs / k;
    const int e = ids[rs];
    for (int c = threadIdx.x; c < K / 8; c += blockDim.x) xs[c] = reinterpret_cast<const uint4*>(x + (size_t)r * K)[c];
    __syncthreads();
    const int j = blockIdx.x * (MV_THREADS / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (j >= I) return;
    const uint4* wg = reinterpret_cast<const uint4*>(W + ((size_t)e * 2 * I + 2 * j) * K);
    const uint4* wu = wg + K / 8;
    float g = 0.f, u = 0.f;
#pragma unroll 4
    for (int c = lane; c < K / 8; c += 32) {
        const uint4 a = ldg_nc_v4(wg + c), b = ldg_nc_v4(wu + c), xv = xs[c];
        const uint32_t* a32 = reinterpret_cast<const uint32_t*>(&a);
        const uint32_t* b32 = reinterpret_cast<const uint32_t*>(&b);
        const uint32_t* x32 = reinterpret_cast<const uint32_t*>(&xv);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            g = fmaf(bf16_lo(a32[q]), bf16_lo(x32[q]), g);
            g = fmaf(bf16_hi(a32[q]), bf16_hi(x32[q]), g);
            u = fmaf(bf16_lo(b32[q]), bf16_lo(x32[q]), u);
            u = fmaf(bf16_hi(b32[q]), bf16_hi(x32[q]), u);
        }
    }
    g = warp_sum(g);
    u = warp_sum(u);
    if (lane == 0) y[(size_t)rs * I + j] = f2bf(rbf(silu_f(rbf(g))) * rbf(u));
}

// grid (ceil(H / 8), M): warp -> output column n of row r; out[r, n] = bf16(residual[r, n] + acc).  Every lane issues
// the loads of all k experts' rows before the first reduction, so a warp keeps k times more bytes in flight than a
// one-expert-at-a-time loop; the k dot products are then reduced and combined in ascending expert order.
__global__ void __launch_bounds__(MV_THREADS)
moe_gemv_down_kernel(const bf16* __restrict__ act, const bf16* __restrict__ W, bf16* __restrict__ out,
                     const int32_t* __restrict__ ids, const float* __restrict__ wts, const bf16* __restrict__ residual,
                     int k, int H, int I) {
    extern __shared__ uint4 as[];
    const int r = blockIdx.y;
    for (int c = threadIdx.x; c < k * I / 8; c += blockDim.x) as[c] = reinterpret_cast<const uint4*>(act + (size_t)r * k * I)[c];
    __syncthreads();
    const int n = blockIdx.x * (MV_THREADS / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (n >= H) return;
    float p[MOE_MAX_K];
    const uint4* w[MOE_MAX_K];
#pragma unroll
    for (int s = 0; s < MOE_MAX_K; ++s) {
        p[s] = 0.f;
        w[s] = s < k ? reinterpret_cast<const uint4*>(W + ((size_t)ids[(size_t)r * k + s] * H + n) * I) : nullptr;
    }
    for (int c = lane; c < I / 8; c += 32) {
        uint4 wv[MOE_MAX_K];
#pragma unroll
        for (int s = 0; s < MOE_MAX_K; ++s)
            if (s < k) wv[s] = ldg_nc_v4(w[s] + c);
#pragma unroll
        for (int s = 0; s < MOE_MAX_K; ++s) {
            if (s < k) {
                const uint4 av = as[s * (I / 8) + c];
                const uint32_t* w32 = reinterpret_cast<const uint32_t*>(&wv[s]);
                const uint32_t* a32 = reinterpret_cast<const uint32_t*>(&av);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    p[s] = fmaf(bf16_lo(w32[q]), bf16_lo(a32[q]), p[s]);
                    p[s] = fmaf(bf16_hi(w32[q]), bf16_hi(a32[q]), p[s]);
                }
            }
        }
    }
    float acc = 0.f;
#pragma unroll
    for (int s = 0; s < MOE_MAX_K; ++s) {
        if (s < k) acc = moe_add(acc, rbf(warp_sum(p[s])), wts[(size_t)r * k + s]);
    }
    if (lane == 0) out[(size_t)r * H + n] = f2bf(bf2f(residual[(size_t)r * H + n]) + acc);
}

}  // namespace tl

using namespace tl;

extern "C" int tl_moe_route(const void* logits, int N, int E, int k, int norm_topk, int32_t* ids, float* wts,
                            int32_t* counts, int32_t* offsets, int32_t* row_of, int32_t* tiles, int max_tiles, void* stream) {
    TL_REQUIRE(N > 0 && E > 0 && E <= MOE_MAX_E && k >= 1 && k <= MOE_MAX_K && k <= E, TL_ERR_INVALID,
               "tl_moe_route: N=%d E=%d k=%d outside N>0, 1<=k<=min(16,E), E<=256", N, E, k);
    const bool plan = counts || offsets || row_of || tiles;
    TL_REQUIRE(!plan || (counts && offsets && row_of && tiles && max_tiles >= tl_moe_max_tiles(N, E, k)), TL_ERR_INVALID,
               "tl_moe_route: the plan needs counts, offsets, row_of and tiles, with max_tiles >= tl_moe_max_tiles");
    cudaStream_t st = (cudaStream_t)stream;
    moe_topk_kernel<<<(N + 7) / 8, 256, 0, st>>>((const bf16*)logits, ids, wts, N, E, k, norm_topk);
    int rc = check_launch("tl_moe_route (top-k)");
    if (rc != TL_OK || !plan) return rc;
    moe_plan_kernel<<<1, MOE_PLAN_THREADS, 0, st>>>(ids, N, E, k, counts, offsets, row_of, tiles, max_tiles);
    return check_launch("tl_moe_route (plan)");
}

extern "C" int tl_moe_max_tiles(int N, int E, int k) {
    const long long picks = (long long)N * k;
    return (int)((picks + BM - 1) / BM + (picks < E ? picks : E));
}

extern "C" int tl_moe_gather(const void* h, const int32_t* row_of, void* hg, int N, int k, int H, void* stream) {
    TL_REQUIRE(N > 0 && k > 0 && H % 8 == 0, TL_ERR_INVALID, "tl_moe_gather: N=%d k=%d H=%d", N, k, H);
    moe_gather_kernel<<<N * k, 256, 0, (cudaStream_t)stream>>>((const bf16*)h, row_of, (bf16*)hg, k, H);
    return check_launch("tl_moe_gather");
}

extern "C" int tl_moe_combine(const void* y, const int32_t* row_of, const float* wts, const void* x, void* out, int N, int k,
                              int H, void* stream) {
    TL_REQUIRE(N > 0 && k > 0 && H % 2 == 0, TL_ERR_INVALID, "tl_moe_combine: N=%d k=%d H=%d", N, k, H);
    moe_combine_kernel<<<N, 256, 0, (cudaStream_t)stream>>>((const bf16*)y, row_of, wts, (const bf16*)x, (bf16*)out, k, H);
    return check_launch("tl_moe_combine");
}

extern "C" int tl_moe_gemm(const void* A, const void* W, void* C, const int32_t* tiles, int max_tiles, int E, int N, int K,
                           int ldc, int flags, void* stream) {
    TL_REQUIRE(max_tiles > 0 && E > 0 && N > 0 && K > 0 && N % MG_BN == 0 && K % 8 == 0, TL_ERR_INVALID,
               "tl_moe_gemm: N=%d must be a multiple of %d and K=%d of 8", N, MG_BN, K);
    TL_REQUIRE(flags == 0 || flags == TL_EPI_SWIGLU, TL_ERR_INVALID, "tl_moe_gemm: flags must be 0 or TL_EPI_SWIGLU");
    TL_REQUIRE(ldc >= ((flags & TL_EPI_SWIGLU) ? N / 2 : N) && ldc % 8 == 0, TL_ERR_INVALID, "tl_moe_gemm: ldc=%d", ldc);
    CUtensorMap tmA, tmB;
    int rc = make_tensor_map(&tmA, A, (uint64_t)K, (uint64_t)max_tiles * BM, (uint64_t)K, BK, BM);
    if (rc != TL_OK) return rc;
    rc = make_tensor_map(&tmB, W, (uint64_t)K, (uint64_t)E * N, (uint64_t)K, BK, MG_BN);
    if (rc != TL_OK) return rc;
    static bool attr_done = false;
    if (!attr_done) {
        if (cudaFuncSetAttribute(moe_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MG_SMEM_BYTES) != cudaSuccess)
            return check_launch("tl_moe_gemm (smem attr)");
        attr_done = true;
    }
    const int total = max_tiles * (N / MG_BN);
    const int grid = total < sm_count() ? total : sm_count();
    moe_gemm_kernel<<<grid, MG_THREADS, MG_SMEM_BYTES, (cudaStream_t)stream>>>(tmA, tmB, (bf16*)C, tiles, max_tiles, N, K, ldc,
                                                                               flags);
    return check_launch("tl_moe_gemm");
}

extern "C" int tl_moe_gemv(const void* x, const void* W, void* y, const int32_t* ids, const float* wts, const void* residual,
                           int M, int k, int N, int K, int flags, void* stream) {
    TL_REQUIRE(M >= 1 && M <= 16 && k >= 1 && k <= MOE_MAX_K && N > 0 && K > 0 && K % 8 == 0, TL_ERR_INVALID,
               "tl_moe_gemv: M=%d k=%d N=%d K=%d", M, k, N, K);
    cudaStream_t st = (cudaStream_t)stream;
    const int wpb = MV_THREADS / 32;
    if (flags == TL_EPI_SWIGLU) {
        TL_REQUIRE(N % 2 == 0 && (size_t)K * 2 <= 48 * 1024, TL_ERR_INVALID, "tl_moe_gemv: SwiGLU needs even N, K <= 24576");
        const int I = N / 2;
        moe_gemv_gu_kernel<<<dim3((I + wpb - 1) / wpb, M * k), MV_THREADS, K * 2, st>>>((const bf16*)x, (const bf16*)W, (bf16*)y,
                                                                                    ids, k, I, K);
        return check_launch("tl_moe_gemv (gate/up)");
    }
    TL_REQUIRE(flags == TL_EPI_RESIDUAL && residual && wts, TL_ERR_INVALID,
               "tl_moe_gemv: flags must be TL_EPI_SWIGLU or TL_EPI_RESIDUAL (down + combine, with wts and residual)");
    TL_REQUIRE((size_t)k * K * 2 <= 48 * 1024, TL_ERR_INVALID, "tl_moe_gemv: k*K=%d too large for the staged rows", k * K);
    moe_gemv_down_kernel<<<dim3((N + wpb - 1) / wpb, M), MV_THREADS, k * K * 2, st>>>(
        (const bf16*)x, (const bf16*)W, (bf16*)y, ids, wts, (const bf16*)residual, k, N, K);
    return check_launch("tl_moe_gemv (down + combine)");
}
