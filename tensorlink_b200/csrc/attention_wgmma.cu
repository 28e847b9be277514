// Causal GQA attention on Hopper tensor cores (wgmma): prefill forward and the two backward passes.
//
// One warpgroup (128 threads) per CTA and 64 rows per tile.  Every operand tile (64 rows x D columns of bf16) arrives by
// TMA as D/64 boxes of 64 x 64 with the 128-byte swizzle, and a two-slot mbarrier ring streams the inner loop's tiles.
// The first product of each step (S = Q·K^T, dP = dO·V^T, ...) accumulates in registers.  Its accumulator fragment has
// the layout of wgmma's register A operand, so P / dS go into the second product (P·V, dS·K, P^T·dO, dS^T·Q) without
// passing through shared memory.  A tile that is K-major for one product is the MN-major operand of the other: K and V
// rows serve S = Q·K^T and, transposed by the descriptor, O += P·V.
// Numerics follow the mma.sync kernels (attention.cu, attention_bwd.cu): fp32 scores and softmax in the log2 domain,
// P and dS rounded to bf16 for their products, fp32 accumulation, lse in natural log.
// q/o/do/dq: [B,S,n_h,d] token-major;  k/v: [B,n_kv,T_max,d];  dk/dv: [B,n_h,T_max,d] (one partial per query head).
#include "gemm_common.cuh"

namespace tl {

constexpr int AW_ROWS = 64, AW_THREADS = 128;
constexpr float AW_LOG2E = 1.4426950408889634f;

template <int D>
struct AwTile {
    static constexpr int BYTES = AW_ROWS * D * 2;   // D/64 boxes of 8 KB
};

// one tile = D/64 boxes (64 columns x 64 rows) of a row-major [rows, cols] tensor map
template <int D>
__device__ __forceinline__ void aw_load(unsigned char* dst, const CUtensorMap* map, uint64_t* bar, int row, int col0) {
#pragma unroll
    for (int c = 0; c < D / 64; ++c) tma_load_2d(dst + c * 8192, map, bar, col0 + 64 * c, row);
}
// K-major operand (rows x D, contraction over D): the kk-th 16-column slice
__device__ __forceinline__ uint64_t aw_kmajor(const unsigned char* tile, int kk) {
    return make_wgmma_desc_sw128(smem_u32(tile) + (uint32_t)((kk >> 2) * 8192 + (kk & 3) * 32), 16, 1024);
}
// MN-major operand (contraction over the 64 rows, N = D columns): the kk-th 16-row slice
__device__ __forceinline__ uint64_t aw_mnmajor(const unsigned char* tile, int kk) {
    return make_wgmma_desc_sw128(smem_u32(tile) + (uint32_t)(kk * 2048), 8192, 1024);
}
// zero rows [valid, 64) of a tile (rows stay whole 128-byte lines under the swizzle); the tile is then read by wgmma
template <int D>
__device__ __forceinline__ void aw_zero_rows(unsigned char* tile, int valid) {
    for (int i = threadIdx.x; i < (D / 64) * AW_ROWS * 8; i += AW_THREADS) {
        const int box = i / (AW_ROWS * 8), rem = i - box * AW_ROWS * 8, row = rem >> 3;
        if (row >= valid) *reinterpret_cast<uint4*>(tile + box * 8192 + row * 128 + (rem & 7) * 16) = make_uint4(0, 0, 0, 0);
    }
    fence_proxy_async();
}
// zero rows [0, lo) and [hi, 64) of a tile: the first KV tile of a left-padded row (pad slots below lo hold anything)
template <int D>
__device__ __forceinline__ void aw_zero_rows_outside(unsigned char* tile, int lo, int hi) {
    for (int i = threadIdx.x; i < (D / 64) * AW_ROWS * 8; i += AW_THREADS) {
        const int box = i / (AW_ROWS * 8), rem = i - box * AW_ROWS * 8, row = rem >> 3;
        if (row < lo || row >= hi) *reinterpret_cast<uint4*>(tile + box * 8192 + row * 128 + (rem & 7) * 16) = make_uint4(0, 0, 0, 0);
    }
    fence_proxy_async();
}

// S (+)= A·B^T over D (both K-major tiles), 64 x 64 fp32 accumulator
template <int D>
__device__ __forceinline__ void aw_qk(float (&s)[32], const unsigned char* a, const unsigned char* b) {
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) wgmma_m64n64<0, 0>(s, aw_kmajor(a, kk), aw_kmajor(b, kk), kk > 0 ? 1u : 0u);
}
// acc += F·T where F (64 x 64) is given as bf16 A fragments and T is a 64 x D tile read MN-major
template <int D>
__device__ __forceinline__ void aw_pv(float (&acc)[D / 2], const uint32_t (&f)[4][4], const unsigned char* t) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        if constexpr (D == 128) wgmma_rs_m64n128<1>(acc, f[kk], aw_mnmajor(t, kk), 1u);
        else wgmma_rs_m64n64<1>(acc, f[kk], aw_mnmajor(t, kk), 1u);
    }
}
// accumulator register i of this thread: row (0..63) and column (0..63)
__device__ __forceinline__ int aw_row(int i) { return 16 * (threadIdx.x >> 5) + ((threadIdx.x & 31) >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int aw_col(int i) { return 8 * (i >> 2) + 2 * (threadIdx.x & 3) + (i & 1); }
// 64 x 64 fp32 values (accumulator layout) -> bf16 A fragments of the four 16-column slices
__device__ __forceinline__ void aw_frag(const float (&v)[32], uint32_t (&f)[4][4]) {
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) f[j][e] = pack_bf16(v[8 * j + 2 * e], v[8 * j + 2 * e + 1]);
}
template <int R>
__device__ __forceinline__ void aw_zero(float (&v)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) v[i] = 0.f;
}

// ================================================================================================ prefill forward
// ROWS: keys below kv_start[b] (left padding of row b) are never attended.  The KV loop starts at tile kv_start / 64,
// and a query tile whose every row sits below kv_start writes zeros (lse = -inf) without loading K/V.
template <int D, bool ROWS>
__global__ void __launch_bounds__(AW_THREADS) attn_fwd_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ,
                                                                    const __grid_constant__ CUtensorMap tmKV_k,
                                                                    const __grid_constant__ CUtensorMap tmKV_v,
                                                                    bf16* __restrict__ out, float* __restrict__ lse, int S,
                                                                    int past_len, int n_h, int n_kv, int T_max, float sl2,
                                                                    const int32_t* __restrict__ kv_start) {
    constexpr int TB = AwTile<D>::BYTES;
    extern __shared__ unsigned char smem_dyn[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    unsigned char* sQ = smem;
    unsigned char* sK = smem + TB;                   // [2] slots, K then V in each
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 5 * TB);   // [0] = Q, [1..2] = K/V slots
    const int q0 = blockIdx.x * AW_ROWS, h = blockIdx.y, b = blockIdx.z, kvh = h / (n_h / n_kv);
    const int T = past_len + S;                          // valid keys
    const int n_keys = min(T, past_len + q0 + AW_ROWS);  // causal limit of this query tile
    const int n_tiles = (n_keys + AW_ROWS - 1) / AW_ROWS;
    const int kv_row = (b * n_kv + kvh) * T_max;
    int k_start = 0, t0 = 0;                                  // first valid key and its tile
    if constexpr (ROWS) {
        k_start = kv_start[b];
        if (n_keys <= k_start) {                              // every query row of this tile is a pad row
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int row = q0 + aw_row(0) + 8 * r;
                if (row >= S) continue;
                bf16* dst = out + ((size_t)b * S + row) * n_h * D + (size_t)h * D;
#pragma unroll
                for (int i = 2 * r; i < D / 2; i += 4) *reinterpret_cast<uint32_t*>(dst + aw_col(i)) = 0u;
                if (lse && (threadIdx.x & 3) == 0) lse[((size_t)b * n_h + h) * S + row] = -INFINITY;
            }
            return;
        }
        t0 = k_start / AW_ROWS;
    }
    if (threadIdx.x == 0) {
        for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
        fence_barrier_init();
        mbar_expect_tx(&bars[0], TB);
        aw_load<D>(sQ, &tmQ, &bars[0], b * S + q0, h * D);
        for (int t = 0; t < 2 && t0 + t < n_tiles; ++t) {
            mbar_expect_tx(&bars[1 + t], 2 * TB);
            aw_load<D>(sK + t * 2 * TB, &tmKV_k, &bars[1 + t], kv_row + (t0 + t) * AW_ROWS, 0);
            aw_load<D>(sK + t * 2 * TB + TB, &tmKV_v, &bars[1 + t], kv_row + (t0 + t) * AW_ROWS, 0);
        }
    }
    __syncthreads();
    mbar_wait(&bars[0], 0);

    float o[D / 2], m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    aw_zero(o);
    const int qpos0 = past_len + q0 + aw_row(0);         // rows aw_row(0) and aw_row(0) + 8
    for (int t = t0; t < n_tiles; ++t) {
        const int slot = (t - t0) & 1;
        unsigned char* k = sK + slot * 2 * TB;
        unsigned char* v = k + TB;
        mbar_wait(&bars[1 + slot], ((t - t0) >> 1) & 1);
        const int kv0 = t * AW_ROWS;
        if constexpr (ROWS) {
            if (kv0 < k_start || kv0 + AW_ROWS > T) {         // pad slots below k_start and rows past T: P·V must see zeros
                aw_zero_rows_outside<D>(v, k_start - kv0, T - kv0);
                __syncthreads();
            }
        } else if (kv0 + AW_ROWS > T) {                  // rows past the valid keys may hold anything: P·V must see zeros
            aw_zero_rows<D>(v, T - kv0);
            __syncthreads();
        }
        float s[32];
        wgmma_fence_acc(s);
        wgmma_fence();
        aw_qk<D>(s, sQ, k);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(s);
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            const int key = kv0 + aw_col(i), r = (i >> 1) & 1;
            float x = s[i] * sl2;
            if (key > qpos0 + 8 * r || key >= T) x = -INFINITY;
            if constexpr (ROWS) if (key < k_start) x = -INFINITY;
            s[i] = x;
            mx[r] = fmaxf(mx[r], x);
        }
        float alpha[2], msub[2], rs[2] = {0.f, 0.f};
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            const float m_new = fmaxf(m_run[r], mx[r]);
            msub[r] = (m_new == -INFINITY) ? 0.f : m_new;
            alpha[r] = exp2f(m_run[r] - msub[r]);
            m_run[r] = m_new;
        }
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            s[i] = exp2f(s[i] - msub[(i >> 1) & 1]);
            rs[(i >> 1) & 1] += s[i];
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 1);
            rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 2);
            l_run[r] = l_run[r] * alpha[r] + rs[r];
        }
#pragma unroll
        for (int i = 0; i < D / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
        uint32_t pf[4][4];
        aw_frag(s, pf);
        wgmma_fence_acc(o);
        wgmma_fence();
        aw_pv<D>(o, pf, v);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(o);
        __syncthreads();                                 // every thread is done with this slot
        if (threadIdx.x == 0 && t + 2 < n_tiles) {
            mbar_expect_tx(&bars[1 + slot], 2 * TB);
            aw_load<D>(k, &tmKV_k, &bars[1 + slot], kv_row + (t + 2) * AW_ROWS, 0);
            aw_load<D>(v, &tmKV_v, &bars[1 + slot], kv_row + (t + 2) * AW_ROWS, 0);
        }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = q0 + aw_row(0) + 8 * r;
        if (row >= S) continue;
        const float inv = l_run[r] > 0.f ? 1.0f / l_run[r] : 0.f;
        bf16* dst = out + ((size_t)b * S + row) * n_h * D + (size_t)h * D;
#pragma unroll
        for (int i = 2 * r; i < D / 2; i += 4) {
            *reinterpret_cast<uint32_t*>(dst + aw_col(i)) = pack_bf16(o[i] * inv, o[i + 1] * inv);
        }
        if (lse && (threadIdx.x & 3) == 0)
            lse[((size_t)b * n_h + h) * S + row] = m_run[r] * 0.6931471805599453f + logf(l_run[r]);
    }
}

// ================================================================================================ backward pass 1: dQ
// ROWS: keys below kv_start[b] are pad slots.  A query tile made only of pad rows writes dq = 0 and loads nothing; the
// KV loop starts at tile kv_start / 64, the first tile's pad K/V rows are zeroed, and P / dS of pad keys (and so of pad
// query rows, which see no key at or below them) are 0 by select: pad q, dO, lse and D may hold anything.
template <int D, bool ROWS>
__global__ void __launch_bounds__(AW_THREADS) attn_bwd_dq_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ,
                                                                       const __grid_constant__ CUtensorMap tmdO,
                                                                       const __grid_constant__ CUtensorMap tmK,
                                                                       const __grid_constant__ CUtensorMap tmV,
                                                                       const float* __restrict__ lse, const float* __restrict__ Dv,
                                                                       bf16* __restrict__ dq, int S, int n_h, int n_kv, int T_max,
                                                                       float scale, const int32_t* __restrict__ kv_start) {
    constexpr int TB = AwTile<D>::BYTES;
    extern __shared__ unsigned char smem_dyn[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    unsigned char* sQ = smem;
    unsigned char* sdO = smem + TB;
    unsigned char* sK = smem + 2 * TB;               // [2] slots, K then V in each
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 6 * TB);
    const int q0 = blockIdx.x * AW_ROWS, h = blockIdx.y, b = blockIdx.z, kvh = h / (n_h / n_kv);
    const int n_keys = min(S, q0 + AW_ROWS);
    const int n_tiles = (n_keys + AW_ROWS - 1) / AW_ROWS;
    const int kv_row = (b * n_kv + kvh) * T_max;
    int k_start = 0, t0 = 0;                                  // first valid key and its tile
    if constexpr (ROWS) {
        k_start = kv_start[b];
        if (n_keys <= k_start) {                              // every query row of this tile is a pad row
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int row = q0 + aw_row(0) + 8 * r;
                if (row >= S) continue;
                bf16* dst = dq + ((size_t)b * S + row) * n_h * D + (size_t)h * D;
#pragma unroll
                for (int i = 2 * r; i < D / 2; i += 4) *reinterpret_cast<uint32_t*>(dst + aw_col(i)) = 0u;
            }
            return;
        }
        t0 = k_start / AW_ROWS;
    }
    if (threadIdx.x == 0) {
        for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
        fence_barrier_init();
        mbar_expect_tx(&bars[0], 2 * TB);
        aw_load<D>(sQ, &tmQ, &bars[0], b * S + q0, h * D);
        aw_load<D>(sdO, &tmdO, &bars[0], b * S + q0, h * D);
        for (int t = 0; t < 2 && t0 + t < n_tiles; ++t) {
            mbar_expect_tx(&bars[1 + t], 2 * TB);
            aw_load<D>(sK + t * 2 * TB, &tmK, &bars[1 + t], kv_row + (t0 + t) * AW_ROWS, 0);
            aw_load<D>(sK + t * 2 * TB + TB, &tmV, &bars[1 + t], kv_row + (t0 + t) * AW_ROWS, 0);
        }
    }
    const int row0 = q0 + aw_row(0);
    float lse2[2], dvr[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = row0 + 8 * r;
        const bool ok = row < S;
        lse2[r] = ok ? lse[((size_t)b * n_h + h) * S + row] * AW_LOG2E : 0.f;
        dvr[r] = ok ? Dv[((size_t)b * n_h + h) * S + row] : 0.f;
    }
    const float sl2 = scale * AW_LOG2E;
    __syncthreads();
    mbar_wait(&bars[0], 0);

    float acc[D / 2];
    aw_zero(acc);
    for (int t = t0; t < n_tiles; ++t) {
        const int slot = (t - t0) & 1;
        unsigned char* k = sK + slot * 2 * TB;
        unsigned char* v = k + TB;
        mbar_wait(&bars[1 + slot], ((t - t0) >> 1) & 1);
        const int kv0 = t * AW_ROWS;
        if constexpr (ROWS) {
            if (kv0 < k_start || kv0 + AW_ROWS > S) {         // pad slots and keys past S: dS = 0 must meet finite K / V
                aw_zero_rows_outside<D>(k, k_start - kv0, S - kv0);
                aw_zero_rows_outside<D>(v, k_start - kv0, S - kv0);
                __syncthreads();
            }
        } else if (kv0 + AW_ROWS > S) {                  // keys past S: dS = 0 must meet finite K / V rows
            aw_zero_rows<D>(k, S - kv0);
            aw_zero_rows<D>(v, S - kv0);
            __syncthreads();
        }
        float s[32], dp[32];
        wgmma_fence_acc(s);
        wgmma_fence_acc(dp);
        wgmma_fence();
        aw_qk<D>(s, sQ, k);
        aw_qk<D>(dp, sdO, v);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(s);
        wgmma_fence_acc(dp);
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            const int key = kv0 + aw_col(i), r = (i >> 1) & 1;
            if constexpr (ROWS) {       // key >= k_start also masks pad query rows (key <= row < k_start)
                const bool ok = key <= row0 + 8 * r && key < S && key >= k_start;
                s[i] = ok ? exp2f(s[i] * sl2 - lse2[r]) * (dp[i] - dvr[r]) * scale : 0.f;
            } else {
                const float p = (key > row0 + 8 * r || key >= S) ? 0.f : exp2f(s[i] * sl2 - lse2[r]);
                s[i] = p * (dp[i] - dvr[r]) * scale;
            }
        }
        uint32_t dsf[4][4];
        aw_frag(s, dsf);
        wgmma_fence_acc(acc);
        wgmma_fence();
        aw_pv<D>(acc, dsf, k);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(acc);
        __syncthreads();
        if (threadIdx.x == 0 && t + 2 < n_tiles) {
            mbar_expect_tx(&bars[1 + slot], 2 * TB);
            aw_load<D>(k, &tmK, &bars[1 + slot], kv_row + (t + 2) * AW_ROWS, 0);
            aw_load<D>(v, &tmV, &bars[1 + slot], kv_row + (t + 2) * AW_ROWS, 0);
        }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = row0 + 8 * r;
        if (row >= S) continue;
        bf16* dst = dq + ((size_t)b * S + row) * n_h * D + (size_t)h * D;
#pragma unroll
        for (int i = 2 * r; i < D / 2; i += 4) *reinterpret_cast<uint32_t*>(dst + aw_col(i)) = pack_bf16(acc[i], acc[i + 1]);
    }
}

// ================================================================================================ backward pass 2: dK, dV
// ROWS: a key tile lying wholly below kv_start[b] writes dk = dv = 0 and loads nothing.  P / dS of pad keys and pad
// query rows are 0 by select, and the Q / dO rows of a query tile outside [kv_start, S) are zeroed before they meet
// P^T / dS^T (rows past S belong to the next batch row and may be its pad rows), so pad key rows end as exact zeros.
template <int D, bool ROWS>
__global__ void __launch_bounds__(AW_THREADS) attn_bwd_dkv_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ,
                                                                        const __grid_constant__ CUtensorMap tmdO,
                                                                        const __grid_constant__ CUtensorMap tmK,
                                                                        const __grid_constant__ CUtensorMap tmV,
                                                                        const float* __restrict__ lse, const float* __restrict__ Dv,
                                                                        bf16* __restrict__ dk, bf16* __restrict__ dv, int S, int n_h,
                                                                        int n_kv, int T_max, float scale,
                                                                        const int32_t* __restrict__ kv_start) {
    constexpr int TB = AwTile<D>::BYTES;
    extern __shared__ unsigned char smem_dyn[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    unsigned char* sK = smem;
    unsigned char* sV = smem + TB;
    unsigned char* sQ = smem + 2 * TB;               // [2] slots, Q then dO in each
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 6 * TB);
    const int k0 = blockIdx.x * AW_ROWS, h = blockIdx.y, b = blockIdx.z, kvh = h / (n_h / n_kv);
    const int qt0 = blockIdx.x, n_tiles = (S + AW_ROWS - 1) / AW_ROWS - qt0;   // query tiles at or after this key tile
    const int kv_row = (b * n_kv + kvh) * T_max;
    int k_start = 0;
    if constexpr (ROWS) {
        k_start = kv_start[b];
        if (k0 + AW_ROWS <= k_start) {                        // every key of this tile is a pad slot
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int key = k0 + aw_row(0) + 8 * r;
                if (key >= S) continue;
                bf16* dkd = dk + (((size_t)b * n_h + h) * T_max + key) * D;
                bf16* dvd = dv + (((size_t)b * n_h + h) * T_max + key) * D;
#pragma unroll
                for (int i = 2 * r; i < D / 2; i += 4) {
                    *reinterpret_cast<uint32_t*>(dkd + aw_col(i)) = 0u;
                    *reinterpret_cast<uint32_t*>(dvd + aw_col(i)) = 0u;
                }
            }
            return;
        }
    }
    if (threadIdx.x == 0) {
        for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
        fence_barrier_init();
        mbar_expect_tx(&bars[0], 2 * TB);
        aw_load<D>(sK, &tmK, &bars[0], kv_row + k0, 0);
        aw_load<D>(sV, &tmV, &bars[0], kv_row + k0, 0);
        for (int t = 0; t < 2 && t < n_tiles; ++t) {
            mbar_expect_tx(&bars[1 + t], 2 * TB);
            aw_load<D>(sQ + t * 2 * TB, &tmQ, &bars[1 + t], b * S + (qt0 + t) * AW_ROWS, h * D);
            aw_load<D>(sQ + t * 2 * TB + TB, &tmdO, &bars[1 + t], b * S + (qt0 + t) * AW_ROWS, h * D);
        }
    }
    const int key0 = k0 + aw_row(0);                     // rows = keys
    const float sl2 = scale * AW_LOG2E;
    const float* lse_bh = lse + ((size_t)b * n_h + h) * S;
    const float* dv_bh = Dv + ((size_t)b * n_h + h) * S;
    __syncthreads();
    mbar_wait(&bars[0], 0);

    float dka[D / 2], dva[D / 2];
    aw_zero(dka);
    aw_zero(dva);
    for (int t = 0; t < n_tiles; ++t) {
        const int slot = t & 1;
        unsigned char* qt = sQ + slot * 2 * TB;
        unsigned char* dot = qt + TB;
        mbar_wait(&bars[1 + slot], (t >> 1) & 1);
        const int qb = (qt0 + t) * AW_ROWS;
        if constexpr (ROWS) {
            if (qb < k_start || qb + AW_ROWS > S) {           // pad query rows and rows past S: P^T·dO, dS^T·Q see zeros
                aw_zero_rows_outside<D>(qt, k_start - qb, S - qb);
                aw_zero_rows_outside<D>(dot, k_start - qb, S - qb);
                __syncthreads();
            }
        }
        float st[32], dpt[32];
        wgmma_fence_acc(st);
        wgmma_fence_acc(dpt);
        wgmma_fence();
        aw_qk<D>(st, sK, qt);                            // S^T = K·Q^T
        aw_qk<D>(dpt, sV, dot);                          // dP^T = V·dO^T
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(st);
        wgmma_fence_acc(dpt);
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            const int qpos = qb + aw_col(i), key = key0 + 8 * ((i >> 1) & 1);
            const bool ok = qpos < S && key <= qpos && (!ROWS || key >= k_start);
            const int qc = min(qpos, S - 1);
            const float p = ok ? exp2f(st[i] * sl2 - lse_bh[qc] * AW_LOG2E) : 0.f;
            st[i] = p;
            dpt[i] = ok ? p * (dpt[i] - dv_bh[qc]) * scale : 0.f;
        }
        uint32_t pf[4][4], dsf[4][4];
        aw_frag(st, pf);
        aw_frag(dpt, dsf);
        wgmma_fence_acc(dva);
        wgmma_fence_acc(dka);
        wgmma_fence();
        aw_pv<D>(dva, pf, dot);                          // dV += P^T·dO
        aw_pv<D>(dka, dsf, qt);                          // dK += dS^T·Q
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(dva);
        wgmma_fence_acc(dka);
        __syncthreads();
        if (threadIdx.x == 0 && t + 2 < n_tiles) {
            mbar_expect_tx(&bars[1 + slot], 2 * TB);
            aw_load<D>(qt, &tmQ, &bars[1 + slot], b * S + (qt0 + t + 2) * AW_ROWS, h * D);
            aw_load<D>(dot, &tmdO, &bars[1 + slot], b * S + (qt0 + t + 2) * AW_ROWS, h * D);
        }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int key = key0 + 8 * r;
        if (key >= S) continue;
        bf16* dkd = dk + (((size_t)b * n_h + h) * T_max + key) * D;
        bf16* dvd = dv + (((size_t)b * n_h + h) * T_max + key) * D;
#pragma unroll
        for (int i = 2 * r; i < D / 2; i += 4) {
            *reinterpret_cast<uint32_t*>(dkd + aw_col(i)) = pack_bf16(dka[i], dka[i + 1]);
            *reinterpret_cast<uint32_t*>(dvd + aw_col(i)) = pack_bf16(dva[i], dva[i + 1]);
        }
    }
}

// ================================================================================================ host
// the shared-memory opt-in of each instantiation, once
template <int D, int WHICH>
static void aw_smem_attr(const void* kern, int bytes) {
    static bool done = false;
    if (!done) { cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes); done = true; }
}

// kv_start (int32[B], device) non-null: the left-padded instantiation (ROWS)
int attn_prefill_wgmma(const void* q, const void* k_cache, const void* v_cache, void* out, float* lse, int B, int S, int past_len,
                       int n_h, int n_kv, int d, int T_max, float scale, const int32_t* kv_start, cudaStream_t st) {
    CUtensorMap tq, tk, tv;
    int rc = make_tensor_map(&tq, q, (uint64_t)n_h * d, (uint64_t)B * S, (uint64_t)n_h * d, 64, 64);
    if (rc == TL_OK) rc = make_tensor_map(&tk, k_cache, d, (uint64_t)B * n_kv * T_max, d, 64, 64);
    if (rc == TL_OK) rc = make_tensor_map(&tv, v_cache, d, (uint64_t)B * n_kv * T_max, d, 64, 64);
    if (rc != TL_OK) return rc;
    const dim3 grid((S + AW_ROWS - 1) / AW_ROWS, n_h, B);
    const float sl2 = scale * AW_LOG2E;
#define TL_AW_FWD(D_, ROWS_, WHICH_)                                                                                        \
    do {                                                                                                                    \
        const int smem = 5 * AwTile<D_>::BYTES + 1024 + 64;                                                                 \
        aw_smem_attr<D_, WHICH_>((const void*)attn_fwd_wgmma_kernel<D_, ROWS_>, smem);                                      \
        attn_fwd_wgmma_kernel<D_, ROWS_><<<grid, AW_THREADS, smem, st>>>(tq, tk, tv, (bf16*)out, lse, S, past_len, n_h, n_kv, \
                                                                         T_max, sl2, kv_start);                             \
    } while (0)
    if (kv_start) {
        if (d == 64) TL_AW_FWD(64, true, 3); else TL_AW_FWD(128, true, 3);
    } else {
        if (d == 64) TL_AW_FWD(64, false, 0); else TL_AW_FWD(128, false, 0);
    }
#undef TL_AW_FWD
    return check_launch("tl_attn_prefill_fwd (wgmma)");
}

// Dv (rowsum dO·O) must already be in place; kv_start (int32[B], device) non-null: the left-padded instantiations (ROWS)
int attn_bwd_wgmma(const void* q, const void* k_cache, const void* v_cache, const void* dout, const float* lse, const float* Dv,
                   void* dq, void* dk, void* dv, int B, int S, int n_h, int n_kv, int d, int T_max, float scale,
                   const int32_t* kv_start, cudaStream_t st) {
    CUtensorMap tq, tdo, tk, tv;
    int rc = make_tensor_map(&tq, q, (uint64_t)n_h * d, (uint64_t)B * S, (uint64_t)n_h * d, 64, 64);
    if (rc == TL_OK) rc = make_tensor_map(&tdo, dout, (uint64_t)n_h * d, (uint64_t)B * S, (uint64_t)n_h * d, 64, 64);
    if (rc == TL_OK) rc = make_tensor_map(&tk, k_cache, d, (uint64_t)B * n_kv * T_max, d, 64, 64);
    if (rc == TL_OK) rc = make_tensor_map(&tv, v_cache, d, (uint64_t)B * n_kv * T_max, d, 64, 64);
    if (rc != TL_OK) return rc;
    const dim3 grid((S + AW_ROWS - 1) / AW_ROWS, n_h, B);
#define TL_AW_BWD(D_, ROWS_, WHICH_)                                                                                        \
    do {                                                                                                                    \
        const int smem = 6 * AwTile<D_>::BYTES + 1024 + 64;                                                                 \
        aw_smem_attr<D_, WHICH_>((const void*)attn_bwd_dq_wgmma_kernel<D_, ROWS_>, smem);                                   \
        aw_smem_attr<D_, WHICH_ + 1>((const void*)attn_bwd_dkv_wgmma_kernel<D_, ROWS_>, smem);                              \
        attn_bwd_dq_wgmma_kernel<D_, ROWS_><<<grid, AW_THREADS, smem, st>>>(tq, tdo, tk, tv, lse, Dv, (bf16*)dq, S, n_h, n_kv, \
                                                                            T_max, scale, kv_start);                        \
        attn_bwd_dkv_wgmma_kernel<D_, ROWS_><<<grid, AW_THREADS, smem, st>>>(tq, tdo, tk, tv, lse, Dv, (bf16*)dk, (bf16*)dv,  \
                                                                             S, n_h, n_kv, T_max, scale, kv_start);         \
    } while (0)
    if (kv_start) {
        if (d == 64) TL_AW_BWD(64, true, 4); else TL_AW_BWD(128, true, 4);
    } else {
        if (d == 64) TL_AW_BWD(64, false, 1); else TL_AW_BWD(128, false, 1);
    }
#undef TL_AW_BWD
    return check_launch("tl_attn_bwd (wgmma)");
}

}  // namespace tl
