// Causal GQA attention (SDPA contract: fp32 scores + softmax, P cast to bf16 for P·V, fp32 accumulate).
//  * prefill / training forward: flash-style, 64-query x 64-key tiles, warp-level mma.sync for query runs shorter than
//    one tile; attention_wgmma.cu serves the rest.
//  * decode: one query per batch row, split over the KV length, HBM-bound on the cache read.
//  * verify: up to 16 consecutive queries of one row at a device-resident position (prompt-lookup decoding), split the
//    same way.
#include <stdlib.h>

#include "common.cuh"

namespace tl {

// ================================================================================================ prefill
constexpr int FA_BQ = 64, FA_BKV = 64, FA_THREADS = 128;

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, bool valid) {
    const uint32_t d = smem_u32(smem_dst);
    const int sz = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldmatrix_x4(uint32_t* r, const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t* r, const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void mma_bf16_16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// ROWS: keys below kv_start[b] (left padding of row b) are never attended: they are zero-filled on load and masked, the
// KV loop starts at tile kv_start / 64, and a query tile whose every row sits below kv_start writes zeros (lse = -inf).
template <int D, bool ROWS>
__global__ void __launch_bounds__(FA_THREADS) attn_prefill_kernel(const bf16* __restrict__ q,
                                                                   const bf16* __restrict__ k_cache,
                                                                   const bf16* __restrict__ v_cache,
                                                                   bf16* __restrict__ out, float* __restrict__ lse,
                                                                   int S, int past_len, int n_h, int n_kv, int T_max,
                                                                   float scale_log2, const int32_t* __restrict__ kv_start) {
    constexpr int LDS = D + 8;   // padded row (elements): conflict-free ldmatrix
    extern __shared__ __align__(16) unsigned char smem_raw[];
    bf16* sQ = reinterpret_cast<bf16*>(smem_raw);          // [64][LDS]
    bf16* sK = sQ + FA_BQ * LDS;                           // [2][64][LDS]
    bf16* sV = sK + 2 * FA_BKV * LDS;                      // [2][64][LDS]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t4 = lane & 3;
    // heavy (late) query tiles first: better tail balance under causal masking
    const int qt = gridDim.x - 1 - blockIdx.x;
    const int h = blockIdx.y, b = blockIdx.z;
    const int kvh = h / (n_h / n_kv);
    const int q0 = qt * FA_BQ;
    const int T = past_len + S;
    const bf16* qg = q + ((size_t)b * S) * n_h * D + (size_t)h * D;
    const bf16* kg = k_cache + ((size_t)b * n_kv + kvh) * T_max * D;
    const bf16* vg = v_cache + ((size_t)b * n_kv + kvh) * T_max * D;
    constexpr int CPR = D / 8;   // 16-byte chunks per row
    int k_start = 0, t0 = 0;                                   // first valid key and its tile
    if constexpr (ROWS) {
        k_start = kv_start[b];
        if (min(T, past_len + q0 + FA_BQ) <= k_start) {        // every query row of this tile is a pad row
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int row = q0 + warp * 16 + g + r * 8;
                if (row >= S) continue;
                bf16* dst = out + ((size_t)b * S + row) * n_h * D + (size_t)h * D;
#pragma unroll
                for (int i = 0; i < D / 8; ++i) *reinterpret_cast<uint32_t*>(dst + i * 8 + 2 * t4) = 0u;
                if (lse && t4 == 0) lse[((size_t)b * n_h + h) * S + row] = -INFINITY;
            }
            return;
        }
        t0 = k_start / FA_BKV;
    }

    for (int c = tid; c < FA_BQ * CPR; c += FA_THREADS) {
        const int r = c / CPR, cc = c - r * CPR;
        const bool ok = (q0 + r) < S;
        cp_async16(sQ + r * LDS + cc * 8, qg + (size_t)(ok ? q0 + r : 0) * n_h * D + cc * 8, ok);
    }
    auto load_kv = [&](int buf, int kv0) {
        for (int c = tid; c < FA_BKV * CPR; c += FA_THREADS) {
            const int r = c / CPR, cc = c - r * CPR;
            const bool ok = (kv0 + r) < T && (!ROWS || (kv0 + r) >= k_start);   // pad slots load as zeros
            const size_t off = (size_t)(ok ? kv0 + r : 0) * D + cc * 8;
            cp_async16(sK + (buf * FA_BKV + r) * LDS + cc * 8, kg + off, ok);
            cp_async16(sV + (buf * FA_BKV + r) * LDS + cc * 8, vg + off, ok);
        }
    };
    const int kv_end = min(T, past_len + q0 + FA_BQ);          // causal upper bound for this query tile
    const int n_tiles = (kv_end + FA_BKV - 1) / FA_BKV;
    load_kv(t0 & 1, t0 * FA_BKV);
    cp_async_commit();

    float o[D / 8][4];
#pragma unroll
    for (int i = 0; i < D / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    uint32_t qf[D / 16][4];
    const int qrow_abs0 = past_len + q0 + warp * 16 + g;       // absolute position of row g (row g+8: +8)

    for (int it = t0; it < n_tiles; ++it) {
        const int buf = it & 1;
        if (it + 1 < n_tiles) load_kv(buf ^ 1, (it + 1) * FA_BKV);
        cp_async_commit();
        cp_async_wait<1>();
        __syncthreads();
        if (it == t0) {
#pragma unroll
            for (int ks = 0; ks < D / 16; ++ks)
                ldmatrix_x4(qf[ks], sQ + (warp * 16 + (lane & 15)) * LDS + ks * 16 + (lane >> 4) * 8);
        }
        const bf16* sKb = sK + buf * FA_BKV * LDS;
        const bf16* sVb = sV + buf * FA_BKV * LDS;
        float s[FA_BKV / 8][4];
#pragma unroll
        for (int i = 0; i < FA_BKV / 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
#pragma unroll
        for (int ks = 0; ks < D / 16; ++ks) {
#pragma unroll
            for (int np = 0; np < FA_BKV / 16; ++np) {
                uint32_t bfr[4];
                const int mi = lane >> 3;
                ldmatrix_x4(bfr, sKb + (np * 16 + (mi >> 1) * 8 + (lane & 7)) * LDS + ks * 16 + (mi & 1) * 8);
                mma_bf16_16816(s[2 * np], qf[ks], bfr[0], bfr[1]);
                mma_bf16_16816(s[2 * np + 1], qf[ks], bfr[2], bfr[3]);
            }
        }
        // ---- scale, causal mask, online softmax (base 2)
        const int kv0 = it * FA_BKV;
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int i = 0; i < FA_BKV / 8; ++i) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = kv0 + i * 8 + 2 * t4 + (e & 1);
                const int qpos = qrow_abs0 + ((e >> 1) ? 8 : 0);
                float v = s[i][e] * scale_log2;
                if (key > qpos || key >= T) v = -INFINITY;
                if constexpr (ROWS) if (key < k_start) v = -INFINITY;
                s[i][e] = v;
                mx[e >> 1] = fmaxf(mx[e >> 1], v);
            }
        }
        float alpha[2], msub[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            const float m_new = fmaxf(m_run[r], mx[r]);
            msub[r] = (m_new == -INFINITY) ? 0.f : m_new;
            alpha[r] = exp2f(m_run[r] - msub[r]);      // m_run = -inf -> 0
            m_run[r] = m_new;
        }
        float rs[2] = {0.f, 0.f};
        uint32_t pf[FA_BKV / 16][4];
#pragma unroll
        for (int i = 0; i < FA_BKV / 8; ++i) {
            const float p0 = exp2f(s[i][0] - msub[0]), p1 = exp2f(s[i][1] - msub[0]);
            const float p2 = exp2f(s[i][2] - msub[1]), p3 = exp2f(s[i][3] - msub[1]);
            rs[0] += p0 + p1;
            rs[1] += p2 + p3;
            pf[i >> 1][(i & 1) * 2] = pack_bf16(p0, p1);
            pf[i >> 1][(i & 1) * 2 + 1] = pack_bf16(p2, p3);
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 1);
            rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 2);
            l_run[r] = l_run[r] * alpha[r] + rs[r];
        }
#pragma unroll
        for (int i = 0; i < D / 8; ++i) {
            o[i][0] *= alpha[0];
            o[i][1] *= alpha[0];
            o[i][2] *= alpha[1];
            o[i][3] *= alpha[1];
        }
        // ---- O += P · V
#pragma unroll
        for (int kk = 0; kk < FA_BKV / 16; ++kk) {
#pragma unroll
            for (int dp = 0; dp < D / 16; ++dp) {
                uint32_t bfr[4];
                const int mi = lane >> 3;
                ldmatrix_x4_trans(bfr, sVb + (kk * 16 + (mi & 1) * 8 + (lane & 7)) * LDS + dp * 16 + (mi >> 1) * 8);
                mma_bf16_16816(o[2 * dp], pf[kk], bfr[0], bfr[1]);
                mma_bf16_16816(o[2 * dp + 1], pf[kk], bfr[2], bfr[3]);
            }
        }
        __syncthreads();
    }
    // ---- normalise and store
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = q0 + warp * 16 + g + r * 8;
        if (row >= S) continue;
        const float inv = l_run[r] > 0.f ? 1.0f / l_run[r] : 0.f;
        bf16* dst = out + ((size_t)b * S + row) * n_h * D + (size_t)h * D;
#pragma unroll
        for (int i = 0; i < D / 8; ++i)
            *reinterpret_cast<uint32_t*>(dst + i * 8 + 2 * t4) = pack_bf16(o[i][2 * r] * inv, o[i][2 * r + 1] * inv);
        if (lse && t4 == 0)
            lse[((size_t)b * n_h + h) * S + row] = m_run[r] * 0.6931471805599453f + logf(l_run[r]);
    }
}

// ================================================================================================ decode
constexpr int DEC_CHUNK = 128, DEC_THREADS = 128, DEC_MAX_REP = 8;
constexpr int DEC_CHUNK_MMA = 256;      // keys per CTA of the tensor-core split kernel (four 64-key tiles through a 2-tile ring)

// partial record per (b, kv head, split): m[REP], l[REP], o[REP][D]  (fp32)
__host__ __device__ inline size_t dec_rec_floats(int n_rep, int D) { return (size_t)n_rep * (2 + D); }

// ROWS: keys below kv_start[b] are never attended; a split wholly below it is not computed (the reduce skips it)
template <int D, bool ROWS>
__global__ void __launch_bounds__(DEC_THREADS) attn_decode_split_kernel(const bf16* __restrict__ q,
                                                                        const bf16* __restrict__ k_cache,
                                                                        const bf16* __restrict__ v_cache,
                                                                        float* __restrict__ ws,
                                                                        const int32_t* __restrict__ kv_len_dev,
                                                                        int n_h, int n_kv, int T_max, int n_splits,
                                                                        float scale_log2, const int32_t* __restrict__ kv_start) {
    const int split = blockIdx.x, kvh = blockIdx.y, b = blockIdx.z;
    const int kv_len = *kv_len_dev;
    const int c0 = split * DEC_CHUNK;
    if (c0 >= kv_len) return;
    int k_start = 0;
    if constexpr (ROWS) {
        k_start = kv_start[b];
        if (c0 + DEC_CHUNK <= k_start) return;
    }
    const int n_rep = n_h / n_kv;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    __shared__ __align__(16) float sq[DEC_MAX_REP][D];
    __shared__ float sp[DEC_MAX_REP][DEC_CHUNK];
    __shared__ float sred[DEC_THREADS / 32][DEC_MAX_REP];
    __shared__ float sm[DEC_MAX_REP];
    __shared__ __align__(16) float so[DEC_THREADS / 32][DEC_MAX_REP][D];

    for (int i = tid; i < n_rep * D; i += DEC_THREADS) {
        const int r = i / D, dd = i - r * D;
        sq[r][dd] = bf2f(q[((size_t)b * n_h + kvh * n_rep + r) * D + dd]);
    }
    __syncthreads();
    // ---- phase A: one key per thread, n_rep dot products
    const int key = c0 + tid;
    const bool valid = key < kv_len && (!ROWS || key >= k_start);
    float sc[DEC_MAX_REP];
#pragma unroll
    for (int r = 0; r < DEC_MAX_REP; ++r) sc[r] = 0.f;
    if (valid) {
        const uint4* kr = reinterpret_cast<const uint4*>(k_cache + (((size_t)b * n_kv + kvh) * T_max + key) * D);
#pragma unroll 4
        for (int c = 0; c < D / 8; ++c) {
            const uint4 kv4 = kr[c];
            const uint32_t* k32 = reinterpret_cast<const uint32_t*>(&kv4);
            float kf[8];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                kf[2 * j] = bf16_lo(k32[j]);
                kf[2 * j + 1] = bf16_hi(k32[j]);
            }
#pragma unroll
            for (int r = 0; r < DEC_MAX_REP; ++r) {
                if (r < n_rep) {
                    const float4 qa = *reinterpret_cast<const float4*>(&sq[r][c * 8]);
                    const float4 qb = *reinterpret_cast<const float4*>(&sq[r][c * 8 + 4]);
                    sc[r] += kf[0] * qa.x + kf[1] * qa.y + kf[2] * qa.z + kf[3] * qa.w + kf[4] * qb.x + kf[5] * qb.y +
                             kf[6] * qb.z + kf[7] * qb.w;
                }
            }
        }
    }
#pragma unroll
    for (int r = 0; r < DEC_MAX_REP; ++r) {
        sc[r] = valid ? sc[r] * scale_log2 : -INFINITY;
        const float mw = warp_max(sc[r]);
        if (lane == 0) sred[warp][r] = mw;
    }
    __syncthreads();
    if (tid < DEC_MAX_REP) {
        float m = sred[0][tid];
#pragma unroll
        for (int w = 1; w < DEC_THREADS / 32; ++w) m = fmaxf(m, sred[w][tid]);
        sm[tid] = m;
    }
    __syncthreads();
    float lsum[DEC_MAX_REP];
#pragma unroll
    for (int r = 0; r < DEC_MAX_REP; ++r) {
        const float p = (valid && r < n_rep) ? exp2f(sc[r] - sm[r]) : 0.f;
        sp[r][tid] = rbf(p);          // P is cast to bf16 before P·V (SDPA contract)
        lsum[r] = warp_sum(p);
    }
    __syncthreads();   // also orders the sred reads above before the writes below
#pragma unroll
    for (int r = 0; r < DEC_MAX_REP; ++r)
        if (lane == 0) sred[warp][r] = lsum[r];
    // ---- phase B: threads own 8 output dims; key groups stride the chunk
    constexpr int TPR = D / 8;                    // threads per V row
    constexpr int KG = DEC_THREADS / TPR;         // key groups
    const int dd0 = (tid % TPR) * 8, kgi = tid / TPR;
    float acc[DEC_MAX_REP][8];
#pragma unroll
    for (int r = 0; r < DEC_MAX_REP; ++r)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[r][j] = 0.f;
    const int nk = min(DEC_CHUNK, kv_len - c0);
    const int k_lo = ROWS ? max(k_start - c0, 0) : 0;           // V rows of pad slots are never read
    for (int kk = k_lo + kgi; kk < nk; kk += KG) {
        const uint4 vv = *reinterpret_cast<const uint4*>(v_cache + (((size_t)b * n_kv + kvh) * T_max + c0 + kk) * D + dd0);
        const uint32_t* v32 = reinterpret_cast<const uint32_t*>(&vv);
        float vf[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            vf[2 * j] = bf16_lo(v32[j]);
            vf[2 * j + 1] = bf16_hi(v32[j]);
        }
#pragma unroll
        for (int r = 0; r < DEC_MAX_REP; ++r) {
            if (r < n_rep) {
                const float p = sp[r][kk];
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[r][j] = fmaf(p, vf[j], acc[r][j]);
            }
        }
    }
    // reduce key groups: first inside the warp (lanes with equal tid % TPR), then across warps through smem
#pragma unroll
    for (int r = 0; r < DEC_MAX_REP; ++r)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float v = acc[r][j];
#pragma unroll
            for (int off = TPR; off < 32; off <<= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
            acc[r][j] = v;
        }
    if (lane < TPR) {
#pragma unroll
        for (int r = 0; r < DEC_MAX_REP; ++r)
            if (r < n_rep) {
#pragma unroll
                for (int j = 0; j < 8; ++j) so[warp][r][dd0 + j] = acc[r][j];
            }
    }
    __syncthreads();
    float* rec = ws + (((size_t)b * n_kv + kvh) * n_splits + split) * dec_rec_floats(n_rep, D);
    for (int i = tid; i < n_rep * D; i += DEC_THREADS) {
        const int r = i / D, dd = i - r * D;
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < DEC_THREADS / 32; ++w) v += so[w][r][dd];
        rec[2 * n_rep + i] = v;
    }
    if (tid < n_rep) {
        float l = 0.f;
#pragma unroll
        for (int w = 0; w < DEC_THREADS / 32; ++w) l += sred[w][tid];
        rec[tid] = sm[tid];
        rec[n_rep + tid] = l;
    }
}

// ---- split phase on tensor cores (mma.sync m16n8k16).  The n_rep query heads that share a kv head are the M rows of
// the MMA (16 rows, the unused ones zero): per cached key the CUDA-core kernel above spends 2 * n_rep * D FMAs plus the
// bf16 unpacking, which at n_rep = 7 is more issue bandwidth than an SM has at its share of the HBM rate.  Here a CTA stages its DEC_CHUNK keys and values in
// shared memory with cp.async (coalesced 16-byte pieces, a ring of two 64-key tiles: the next tile is in flight while one
// is used; DEC_CHUNK_MMA = 256 keys per CTA), each of the 4 warps owns 16 keys of every 64-key tile with its own online-softmax state, and the 4 states are merged
// through shared memory into the (m, l, o) record the reduce kernel below expects.
template <int D, bool ROWS>
__global__ void __launch_bounds__(FA_THREADS) attn_decode_mma_kernel(const bf16* __restrict__ q, const bf16* __restrict__ k_cache,
                                                                      const bf16* __restrict__ v_cache, float* __restrict__ ws,
                                                                      const int32_t* __restrict__ kv_len_dev, int n_h, int n_kv,
                                                                      int T_max, int n_splits, float scale_log2,
                                                                      const int32_t* __restrict__ kv_start) {
    constexpr int LDS = D + 8;
    constexpr int CPR = D / 8;
    constexpr int NT = 2;                                  // shared-memory ring: two 64-key tiles
    const int split = blockIdx.x, kvh = blockIdx.y, b = blockIdx.z;
    const int kv_len = *kv_len_dev;
    const int c0 = split * DEC_CHUNK_MMA;
    if (c0 >= kv_len) return;
    int k_start = 0, t0 = 0;                               // ROWS: first valid key, first tile of this split holding one
    if constexpr (ROWS) {
        k_start = kv_start[b];
        if (c0 + DEC_CHUNK_MMA <= k_start) return;         // wholly below the start: the reduce skips this split
        t0 = max(k_start - c0, 0) / FA_BKV;
    }
    const int n_rep = n_h / n_kv;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    bf16* sQ = reinterpret_cast<bf16*>(smem_raw);          // [16][LDS]
    bf16* sK = sQ + 16 * LDS;                              // [NT][64][LDS]
    bf16* sV = sK + NT * FA_BKV * LDS;                     // [NT][64][LDS]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t4 = lane & 3;
    const bf16* kg = k_cache + ((size_t)b * n_kv + kvh) * T_max * D;
    const bf16* vg = v_cache + ((size_t)b * n_kv + kvh) * T_max * D;
    const bf16* qg = q + ((size_t)b * n_h + kvh * n_rep) * D;
    for (int c = tid; c < 16 * CPR; c += FA_THREADS) {
        const int r = c / CPR, cc = c - r * CPR;
        cp_async16(sQ + r * LDS + cc * 8, qg + (size_t)(r < n_rep ? r : 0) * D + cc * 8, r < n_rep);
    }
    const int n_tiles = min(DEC_CHUNK_MMA / FA_BKV, (kv_len - c0 + FA_BKV - 1) / FA_BKV);
    auto load_tile = [&](int t) {
        const int kv0 = c0 + t * FA_BKV, buf = t & 1;
        for (int c = tid; c < FA_BKV * CPR; c += FA_THREADS) {
            const int r = c / CPR, cc = c - r * CPR;
            const bool ok = (kv0 + r) < kv_len && (!ROWS || (kv0 + r) >= k_start);   // pad slots load as zeros
            const size_t off = (size_t)(ok ? kv0 + r : 0) * D + cc * 8;
            cp_async16(sK + (buf * FA_BKV + r) * LDS + cc * 8, kg + off, ok);
            cp_async16(sV + (buf * FA_BKV + r) * LDS + cc * 8, vg + off, ok);
        }
        cp_async_commit();                                  // (the q rows ride in the first group)
    };
    load_tile(t0);
    if (t0 + 1 < n_tiles) load_tile(t0 + 1);
    float o[D / 8][4];
#pragma unroll
    for (int i = 0; i < D / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    uint32_t qf[D / 16][4];
    for (int t = t0; t < n_tiles; ++t) {
        if (t + 1 < n_tiles) cp_async_wait<1>(); else cp_async_wait<0>();     // tile t has landed (t+1 may be in flight)
        __syncthreads();
        if (t == t0) {
#pragma unroll
            for (int ks = 0; ks < D / 16; ++ks)
                ldmatrix_x4(qf[ks], sQ + (lane & 15) * LDS + ks * 16 + (lane >> 4) * 8);
        }
        const bf16* sKb = sK + ((t & 1) * FA_BKV + warp * 16) * LDS;     // this warp's 16 keys of the tile
        const bf16* sVb = sV + ((t & 1) * FA_BKV + warp * 16) * LDS;
        float sc[2][4];
#pragma unroll
        for (int i = 0; i < 2; ++i) sc[i][0] = sc[i][1] = sc[i][2] = sc[i][3] = 0.f;
#pragma unroll
        for (int ks = 0; ks < D / 16; ++ks) {
            uint32_t bfr[4];
            const int mi = lane >> 3;
            ldmatrix_x4(bfr, sKb + ((mi >> 1) * 8 + (lane & 7)) * LDS + ks * 16 + (mi & 1) * 8);
            mma_bf16_16816(sc[0], qf[ks], bfr[0], bfr[1]);
            mma_bf16_16816(sc[1], qf[ks], bfr[2], bfr[3]);
        }
        const int key0 = c0 + t * FA_BKV + warp * 16;
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = key0 + i * 8 + 2 * t4 + (e & 1);
                const float v = (key < kv_len && (!ROWS || key >= k_start)) ? sc[i][e] * scale_log2 : -INFINITY;
                sc[i][e] = v;
                mx[e >> 1] = fmaxf(mx[e >> 1], v);
            }
        float alpha[2], msub[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            const float m_new = fmaxf(m_run[r], mx[r]);
            msub[r] = (m_new == -INFINITY) ? 0.f : m_new;
            alpha[r] = exp2f(m_run[r] - msub[r]);
            m_run[r] = m_new;
        }
        float rs[2] = {0.f, 0.f};
        uint32_t pf[4];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const float p0 = exp2f(sc[i][0] - msub[0]), p1 = exp2f(sc[i][1] - msub[0]);
            const float p2 = exp2f(sc[i][2] - msub[1]), p3 = exp2f(sc[i][3] - msub[1]);
            rs[0] += p0 + p1;
            rs[1] += p2 + p3;
            pf[i * 2] = pack_bf16(p0, p1);                  // P is cast to bf16 before P.V (SDPA contract); l keeps fp32
            pf[i * 2 + 1] = pack_bf16(p2, p3);
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 1);
            rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 2);
            l_run[r] = l_run[r] * alpha[r] + rs[r];
        }
#pragma unroll
        for (int i = 0; i < D / 8; ++i) {
            o[i][0] *= alpha[0];
            o[i][1] *= alpha[0];
            o[i][2] *= alpha[1];
            o[i][3] *= alpha[1];
        }
#pragma unroll
        for (int dp = 0; dp < D / 16; ++dp) {
            uint32_t bfr[4];
            const int mi = lane >> 3;
            ldmatrix_x4_trans(bfr, sVb + ((mi & 1) * 8 + (lane & 7)) * LDS + dp * 16 + (mi >> 1) * 8);
            mma_bf16_16816(o[2 * dp], pf, bfr[0], bfr[1]);
            mma_bf16_16816(o[2 * dp + 1], pf, bfr[2], bfr[3]);
        }
        if (t + 2 < n_tiles) {
            __syncthreads();                                // every warp is done with this buffer
            load_tile(t + 2);
        }
    }
    // ---- merge the 4 warps' states (rows g and g+8 of each thread) through shared memory; only rows < n_rep matter
    __syncthreads();                                        // everyone is done with the K / V tiles
    float* sM = reinterpret_cast<float*>(sK);               // [4][16]
    float* sL = sM + 64;                                    // [4][16]
    float* sO = sL + 64;                                    // [4][16][D]
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = g + r * 8;
        if (t4 == 0) { sM[warp * 16 + row] = m_run[r]; sL[warp * 16 + row] = l_run[r]; }
#pragma unroll
        for (int i = 0; i < D / 8; ++i) {
            sO[(warp * 16 + row) * D + i * 8 + 2 * t4] = o[i][2 * r];
            sO[(warp * 16 + row) * D + i * 8 + 2 * t4 + 1] = o[i][2 * r + 1];
        }
    }
    __syncthreads();
    float* rec = ws + (((size_t)b * n_kv + kvh) * n_splits + split) * dec_rec_floats(n_rep, D);
    for (int i = tid; i < n_rep * D; i += FA_THREADS) {
        const int r = i / D, dd = i - r * D;
        const float m = fmaxf(fmaxf(sM[r], sM[16 + r]), fmaxf(sM[32 + r], sM[48 + r]));
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < 4; ++w) {
            const float mw = sM[w * 16 + r];
            if (mw != -INFINITY) v += sO[(w * 16 + r) * D + dd] * exp2f(mw - m);
        }
        rec[2 * n_rep + i] = v;
    }
    if (tid < n_rep) {
        const int r = tid;
        const float m = fmaxf(fmaxf(sM[r], sM[16 + r]), fmaxf(sM[32 + r], sM[48 + r]));
        float l = 0.f;
#pragma unroll
        for (int w = 0; w < 4; ++w) {
            const float mw = sM[w * 16 + r];
            if (mw != -INFINITY) l += sL[w * 16 + r] * exp2f(mw - m);
        }
        rec[r] = m;
        rec[n_rep + r] = l;
    }
}

// ROWS: the splits wholly below kv_start[b] were not computed and are not read
template <int D, bool ROWS>
__global__ void attn_decode_reduce_kernel(const float* __restrict__ ws, bf16* __restrict__ out,
                                          const int32_t* __restrict__ kv_len_dev, int n_h, int n_kv, int n_splits, int chunk,
                                          const int32_t* __restrict__ kv_start) {
    const int h = blockIdx.x, b = blockIdx.y, dd = threadIdx.x;
    const int n_rep = n_h / n_kv, kvh = h / n_rep, r = h - kvh * n_rep;
    const int kv_len = *kv_len_dev;
    const int ns = min(n_splits, (kv_len + chunk - 1) / chunk);
    const int s0 = ROWS ? kv_start[b] / chunk : 0;
    const float* base = ws + ((size_t)b * n_kv + kvh) * n_splits * dec_rec_floats(n_rep, D);
    float M = -INFINITY;
    for (int s = s0; s < ns; ++s) M = fmaxf(M, base[s * dec_rec_floats(n_rep, D) + r]);
    float L = 0.f, O = 0.f;
    for (int s = s0; s < ns; ++s) {
        const float* rec = base + s * dec_rec_floats(n_rep, D);
        const float w = exp2f(rec[r] - M);
        L += rec[n_rep + r] * w;
        O += rec[2 * n_rep + r * D + dd] * w;
    }
    out[((size_t)b * n_h + h) * D + dd] = f2bf(L > 0.f ? O / L : 0.f);
}

// ---- verify: q_len <= 16 query tokens of ONE cache row at slots pos..pos+q_len-1 (their keys and values are already
// appended), query i attending to keys 0..pos+i.  The idea of attn_decode_mma_kernel carries over: the (query token,
// head of the GQA group) pairs m = i * n_rep + r are the M rows of mma.sync, n_rep * q_len <= 128 of them, 64 per CTA
// (grid.z = 2 when there are more: the second CTA re-reads the split's K/V through L2).  Each of the 4 warps owns 16 rows
// and every key of a 64-key tile; a CTA covers DEC_CHUNK_MMA keys through the same 2-tile cp.async ring.  Keys at or
// above pos + q_len are never loaded (zero-filled), keys above pos + i are masked out of row i, so whatever the cache
// holds there (stale drafts, NaN) never reaches an output.  Partial record per (kv head, split, row m): m, l, o[D].
constexpr int VER_MAX_Q = 16;

template <int D>
__global__ void __launch_bounds__(FA_THREADS) attn_verify_mma_kernel(const bf16* __restrict__ q, const bf16* __restrict__ k_cache,
                                                                      const bf16* __restrict__ v_cache, float* __restrict__ ws,
                                                                      const int32_t* __restrict__ pos_dev, int q_len, int n_h,
                                                                      int n_kv, int T_max, int n_splits, float scale_log2) {
    constexpr int LDS = D + 8;
    constexpr int CPR = D / 8;
    const int split = blockIdx.x, kvh = blockIdx.y, m0 = blockIdx.z * FA_BQ;
    const int pos = *pos_dev;
    const int kv_total = min(pos + q_len, T_max);
    const int c0 = split * DEC_CHUNK_MMA;
    if (c0 >= kv_total) return;
    const int n_rep = n_h / n_kv, M = n_rep * q_len;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    bf16* sQ = reinterpret_cast<bf16*>(smem_raw);          // [64][LDS]
    bf16* sK = sQ + FA_BQ * LDS;                           // [2][64][LDS]
    bf16* sV = sK + 2 * FA_BKV * LDS;                      // [2][64][LDS]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t4 = lane & 3;
    const bf16* kg = k_cache + (size_t)kvh * T_max * D;
    const bf16* vg = v_cache + (size_t)kvh * T_max * D;
    for (int c = tid; c < FA_BQ * CPR; c += FA_THREADS) {
        const int r = c / CPR, cc = c - r * CPR, m = m0 + r;
        const bool ok = m < M;
        const int i = ok ? m / n_rep : 0, h = kvh * n_rep + (ok ? m - i * n_rep : 0);
        cp_async16(sQ + r * LDS + cc * 8, q + ((size_t)i * n_h + h) * D + cc * 8, ok);
    }
    const int n_tiles = min(DEC_CHUNK_MMA / FA_BKV, (kv_total - c0 + FA_BKV - 1) / FA_BKV);
    auto load_tile = [&](int t) {
        const int kv0 = c0 + t * FA_BKV, buf = t & 1;
        for (int c = tid; c < FA_BKV * CPR; c += FA_THREADS) {
            const int r = c / CPR, cc = c - r * CPR;
            const bool ok = (kv0 + r) < kv_total;
            const size_t off = (size_t)(ok ? kv0 + r : 0) * D + cc * 8;
            cp_async16(sK + (buf * FA_BKV + r) * LDS + cc * 8, kg + off, ok);
            cp_async16(sV + (buf * FA_BKV + r) * LDS + cc * 8, vg + off, ok);
        }
        cp_async_commit();                                  // (the q rows ride in the first group)
    };
    load_tile(0);
    if (1 < n_tiles) load_tile(1);
    const bool active = m0 + warp * 16 < M;                 // a warp whose 16 rows are all padding only loads
    int last[2];                                            // last key of rows g and g+8 (-1: padding row)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int m = m0 + warp * 16 + g + r * 8;
        last[r] = m < M ? min(pos + m / n_rep, kv_total - 1) : -1;
    }
    float o[D / 8][4];
#pragma unroll
    for (int i = 0; i < D / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    uint32_t qf[D / 16][4];
    for (int t = 0; t < n_tiles; ++t) {
        if (t + 1 < n_tiles) cp_async_wait<1>(); else cp_async_wait<0>();
        __syncthreads();
        if (active) {
            if (t == 0) {
#pragma unroll
                for (int ks = 0; ks < D / 16; ++ks)
                    ldmatrix_x4(qf[ks], sQ + (warp * 16 + (lane & 15)) * LDS + ks * 16 + (lane >> 4) * 8);
            }
            const bf16* sKb = sK + (t & 1) * FA_BKV * LDS;
            const bf16* sVb = sV + (t & 1) * FA_BKV * LDS;
            float s[FA_BKV / 8][4];
#pragma unroll
            for (int i = 0; i < FA_BKV / 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
#pragma unroll
            for (int ks = 0; ks < D / 16; ++ks) {
#pragma unroll
                for (int np = 0; np < FA_BKV / 16; ++np) {
                    uint32_t bfr[4];
                    const int mi = lane >> 3;
                    ldmatrix_x4(bfr, sKb + (np * 16 + (mi >> 1) * 8 + (lane & 7)) * LDS + ks * 16 + (mi & 1) * 8);
                    mma_bf16_16816(s[2 * np], qf[ks], bfr[0], bfr[1]);
                    mma_bf16_16816(s[2 * np + 1], qf[ks], bfr[2], bfr[3]);
                }
            }
            const int kv0 = c0 + t * FA_BKV;
            float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
            for (int i = 0; i < FA_BKV / 8; ++i) {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int key = kv0 + i * 8 + 2 * t4 + (e & 1);
                    const float v = key <= last[e >> 1] ? s[i][e] * scale_log2 : -INFINITY;
                    s[i][e] = v;
                    mx[e >> 1] = fmaxf(mx[e >> 1], v);
                }
            }
            float alpha[2], msub[2];
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
                mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
                const float m_new = fmaxf(m_run[r], mx[r]);
                msub[r] = (m_new == -INFINITY) ? 0.f : m_new;
                alpha[r] = exp2f(m_run[r] - msub[r]);
                m_run[r] = m_new;
            }
            float rs[2] = {0.f, 0.f};
            uint32_t pf[FA_BKV / 16][4];
#pragma unroll
            for (int i = 0; i < FA_BKV / 8; ++i) {
                const float p0 = exp2f(s[i][0] - msub[0]), p1 = exp2f(s[i][1] - msub[0]);
                const float p2 = exp2f(s[i][2] - msub[1]), p3 = exp2f(s[i][3] - msub[1]);
                rs[0] += p0 + p1;
                rs[1] += p2 + p3;
                pf[i >> 1][(i & 1) * 2] = pack_bf16(p0, p1);          // P is cast to bf16 before P.V (SDPA contract)
                pf[i >> 1][(i & 1) * 2 + 1] = pack_bf16(p2, p3);
            }
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 1);
                rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 2);
                l_run[r] = l_run[r] * alpha[r] + rs[r];
            }
#pragma unroll
            for (int i = 0; i < D / 8; ++i) {
                o[i][0] *= alpha[0];
                o[i][1] *= alpha[0];
                o[i][2] *= alpha[1];
                o[i][3] *= alpha[1];
            }
#pragma unroll
            for (int kk = 0; kk < FA_BKV / 16; ++kk) {
#pragma unroll
                for (int dp = 0; dp < D / 16; ++dp) {
                    uint32_t bfr[4];
                    const int mi = lane >> 3;
                    ldmatrix_x4_trans(bfr, sVb + (kk * 16 + (mi & 1) * 8 + (lane & 7)) * LDS + dp * 16 + (mi >> 1) * 8);
                    mma_bf16_16816(o[2 * dp], pf[kk], bfr[0], bfr[1]);
                    mma_bf16_16816(o[2 * dp + 1], pf[kk], bfr[2], bfr[3]);
                }
            }
        }
        if (t + 2 < n_tiles) {
            __syncthreads();                                // every warp is done with this buffer
            load_tile(t + 2);
        }
    }
    if (!active) return;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int m = m0 + warp * 16 + g + r * 8;
        if (m >= M) continue;
        float* rec = ws + (((size_t)kvh * n_splits + split) * M + m) * (2 + D);
        if (t4 == 0) { rec[0] = m_run[r]; rec[1] = l_run[r]; }
#pragma unroll
        for (int i = 0; i < D / 8; ++i)
            *reinterpret_cast<float2*>(rec + 2 + i * 8 + 2 * t4) = make_float2(o[i][2 * r], o[i][2 * r + 1]);
    }
}

// one CTA per (query head, query token): merges the splits that hold keys 0..pos+i (the later splits were computed for
// the later tokens only and are not read)
template <int D>
__global__ void attn_verify_reduce_kernel(const float* __restrict__ ws, bf16* __restrict__ out, const int32_t* __restrict__ pos_dev,
                                          int q_len, int n_h, int n_kv, int T_max, int n_splits) {
    const int h = blockIdx.x, i = blockIdx.y, dd = threadIdx.x;
    const int n_rep = n_h / n_kv, kvh = h / n_rep, M = n_rep * q_len, m = i * n_rep + (h - kvh * n_rep);
    const int last = min(*pos_dev + i, T_max - 1);
    const int ns = min(n_splits, last / DEC_CHUNK_MMA + 1);
    const float* base = ws + ((size_t)kvh * n_splits * M + m) * (2 + D);
    const size_t step = (size_t)M * (2 + D);
    float Mx = -INFINITY;
    for (int s = 0; s < ns; ++s) Mx = fmaxf(Mx, base[s * step]);
    float L = 0.f, O = 0.f;
    for (int s = 0; s < ns; ++s) {
        const float* rec = base + s * step;
        if (rec[0] == -INFINITY) continue;
        const float w = exp2f(rec[0] - Mx);
        L += rec[1] * w;
        O += rec[2 + dd] * w;
    }
    out[((size_t)i * n_h + h) * D + dd] = f2bf(L > 0.f ? O / L : 0.f);
}

}  // namespace tl

namespace tl {
int attn_prefill_wgmma(const void* q, const void* k_cache, const void* v_cache, void* out, float* lse, int B, int S, int past_len,
                       int n_h, int n_kv, int d, int T_max, float scale, const int32_t* kv_start, cudaStream_t st);

// kv_start (int32[B], device) non-null: the left-padded instantiations (ROWS)
static int attn_prefill_launch(const void* q, const void* k_cache, const void* v_cache, void* out, float* lse, int B, int S,
                               int past_len, int n_h, int n_kv, int d, int T_max, float scale, const int32_t* kv_start,
                               cudaStream_t st, const char* what) {
    TL_REQUIRE(d == 64 || d == 128, TL_ERR_INVALID, "%s: head_dim %d not in {64,128}", what, d);
    TL_REQUIRE(n_kv > 0 && n_h % n_kv == 0, TL_ERR_INVALID, "%s: n_h %% n_kv != 0", what);
    TL_REQUIRE(past_len >= 0 && past_len + S <= T_max, TL_ERR_INVALID,
               "%s: past_len %d + S %d exceeds cache T_max %d", what, past_len, S, T_max);
    if (B == 0 || S == 0) return TL_OK;
    {   // wgmma kernel (attention_wgmma.cu) from one full 64-row query tile upwards; TL_ATTN_IMPL=mma|wgmma forces a path
        const char* e = getenv("TL_ATTN_IMPL");          // read per call: tests flip it
        const int impl = !e ? 0 : (e[0] == 'm' ? 1 : (e[0] == 'w' ? 2 : 0));
        if (impl == 2 || (impl == 0 && S >= FA_BQ))
            return attn_prefill_wgmma(q, k_cache, v_cache, out, lse, B, S, past_len, n_h, n_kv, d, T_max, scale, kv_start, st);
    }
    const dim3 grid((S + FA_BQ - 1) / FA_BQ, n_h, B);
    const float sl2 = scale * 1.4426950408889634f;
    const size_t smem = (size_t)(FA_BQ + 4 * FA_BKV) * (d + 8) * sizeof(bf16);
#define TL_FA_FWD(D_, ROWS_)                                                                                                \
    do {                                                                                                                    \
        static bool done = false;                                                                                           \
        if (!done) { cudaFuncSetAttribute(attn_prefill_kernel<D_, ROWS_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); done = true; } \
        attn_prefill_kernel<D_, ROWS_><<<grid, FA_THREADS, smem, st>>>((const bf16*)q, (const bf16*)k_cache, (const bf16*)v_cache, \
                                                                        (bf16*)out, lse, S, past_len, n_h, n_kv, T_max, sl2, kv_start); \
    } while (0)
    if (kv_start) {
        if (d == 64) TL_FA_FWD(64, true); else TL_FA_FWD(128, true);
    } else {
        if (d == 64) TL_FA_FWD(64, false); else TL_FA_FWD(128, false);
    }
#undef TL_FA_FWD
    return check_launch(what);
}

static int attn_decode_launch(const void* q, const void* k_cache, const void* v_cache, void* out, const int32_t* kv_len_dev,
                              void* workspace, size_t ws_bytes, int B, int n_h, int n_kv, int d, int T_max, float scale,
                              const int32_t* kv_start, cudaStream_t st, const char* what);
}  // namespace tl

extern "C" {

int tl_attn_prefill_fwd(const void* q, const void* k_cache, const void* v_cache, void* out, float* lse, int B, int S,
                        int past_len, int n_h, int n_kv, int d, int T_max, float scale, void* stream) {
    return tl::attn_prefill_launch(q, k_cache, v_cache, out, lse, B, S, past_len, n_h, n_kv, d, T_max, scale, nullptr,
                                   (cudaStream_t)stream, "tl_attn_prefill_fwd");
}

int tl_attn_prefill_fwd_rows(const void* q, const void* k_cache, const void* v_cache, void* out, float* lse, int B, int S,
                             int past_len, int n_h, int n_kv, int d, int T_max, float scale, const int32_t* kv_start_dev,
                             void* stream) {
    using namespace tl;
    TL_REQUIRE(kv_start_dev != nullptr, TL_ERR_INVALID, "tl_attn_prefill_fwd_rows: kv_start_dev is null");
    return attn_prefill_launch(q, k_cache, v_cache, out, lse, B, S, past_len, n_h, n_kv, d, T_max, scale, kv_start_dev,
                               (cudaStream_t)stream, "tl_attn_prefill_fwd_rows");
}

size_t tl_attn_decode_ws(int B, int n_h, int d, int T_max) {
    const size_t n_splits = (size_t)(T_max + tl::DEC_CHUNK - 1) / tl::DEC_CHUNK;
    return (size_t)B * n_splits * (size_t)n_h * (2 + d) * sizeof(float);
}

int tl_attn_decode_fwd(const void* q, const void* k_cache, const void* v_cache, void* out, const int32_t* kv_len_dev,
                       void* workspace, size_t ws_bytes, int B, int n_h, int n_kv, int d, int T_max, float scale,
                       void* stream) {
    return tl::attn_decode_launch(q, k_cache, v_cache, out, kv_len_dev, workspace, ws_bytes, B, n_h, n_kv, d, T_max, scale,
                                  nullptr, (cudaStream_t)stream, "tl_attn_decode_fwd");
}

int tl_attn_decode_fwd_rows(const void* q, const void* k_cache, const void* v_cache, void* out, const int32_t* kv_len_dev,
                            void* workspace, size_t ws_bytes, int B, int n_h, int n_kv, int d, int T_max, float scale,
                            const int32_t* kv_start_dev, void* stream) {
    using namespace tl;
    TL_REQUIRE(kv_start_dev != nullptr, TL_ERR_INVALID, "tl_attn_decode_fwd_rows: kv_start_dev is null");
    return attn_decode_launch(q, k_cache, v_cache, out, kv_len_dev, workspace, ws_bytes, B, n_h, n_kv, d, T_max, scale,
                              kv_start_dev, (cudaStream_t)stream, "tl_attn_decode_fwd_rows");
}

size_t tl_attn_verify_ws(int q_len, int n_h, int d, int T_max) {
    const size_t n_splits = (size_t)(T_max + tl::DEC_CHUNK_MMA - 1) / tl::DEC_CHUNK_MMA;
    return n_splits * (size_t)n_h * (size_t)(q_len > 0 ? q_len : 0) * (2 + d) * sizeof(float);
}

int tl_attn_verify_fwd(const void* q, const void* k_cache, const void* v_cache, void* out, const int32_t* pos_dev,
                       void* workspace, size_t ws_bytes, int q_len, int n_h, int n_kv, int d, int T_max, float scale,
                       void* stream) {
    using namespace tl;
    const char* what = "tl_attn_verify_fwd";
    TL_REQUIRE(d == 64 || d == 128, TL_ERR_INVALID, "%s: head_dim %d not in {64,128}", what, d);
    TL_REQUIRE(n_kv > 0 && n_h % n_kv == 0 && n_h / n_kv <= DEC_MAX_REP, TL_ERR_INVALID,
               "%s: GQA group %d/%d unsupported (max %d)", what, n_h, n_kv, DEC_MAX_REP);
    TL_REQUIRE(q_len >= 1 && q_len <= VER_MAX_Q, TL_ERR_INVALID, "%s: q_len %d not in [1, %d]", what, q_len, VER_MAX_Q);
    TL_REQUIRE(q && k_cache && v_cache && out && pos_dev && workspace, TL_ERR_INVALID, "%s: null argument", what);
    TL_REQUIRE(T_max >= q_len, TL_ERR_INVALID, "%s: T_max %d < q_len %d", what, T_max, q_len);
    TL_REQUIRE(ws_bytes >= tl_attn_verify_ws(q_len, n_h, d, T_max), TL_ERR_WORKSPACE,
               "%s: workspace %zu < %zu", what, ws_bytes, tl_attn_verify_ws(q_len, n_h, d, T_max));
    const int n_splits = (T_max + DEC_CHUNK_MMA - 1) / DEC_CHUNK_MMA;
    const int M = n_h / n_kv * q_len;
    const dim3 g1(n_splits, n_kv, (M + FA_BQ - 1) / FA_BQ), g2(n_h, q_len);
    const float sl2 = scale * 1.4426950408889634f;
    const size_t smem = (size_t)(FA_BQ + 4 * FA_BKV) * (d + 8) * sizeof(bf16);
    cudaStream_t st = (cudaStream_t)stream;
#define TL_VERIFY(D_)                                                                                                       \
    do {                                                                                                                    \
        static bool done = false;                                                                                           \
        if (!done) { cudaFuncSetAttribute(attn_verify_mma_kernel<D_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); done = true; } \
        attn_verify_mma_kernel<D_><<<g1, FA_THREADS, smem, st>>>((const bf16*)q, (const bf16*)k_cache, (const bf16*)v_cache,     \
                                                                 (float*)workspace, pos_dev, q_len, n_h, n_kv, T_max, n_splits, sl2); \
        attn_verify_reduce_kernel<D_><<<g2, D_, 0, st>>>((const float*)workspace, (bf16*)out, pos_dev, q_len, n_h, n_kv, T_max, \
                                                         n_splits);                                                         \
    } while (0)
    if (d == 64) TL_VERIFY(64); else TL_VERIFY(128);
#undef TL_VERIFY
    return check_launch(what);
}

}  // extern "C"

namespace tl {
static int attn_decode_launch(const void* q, const void* k_cache, const void* v_cache, void* out, const int32_t* kv_len_dev,
                              void* workspace, size_t ws_bytes, int B, int n_h, int n_kv, int d, int T_max, float scale,
                              const int32_t* kv_start, cudaStream_t st, const char* what) {
    TL_REQUIRE(d == 64 || d == 128, TL_ERR_INVALID, "%s: head_dim %d not in {64,128}", what, d);
    TL_REQUIRE(n_kv > 0 && n_h % n_kv == 0 && n_h / n_kv <= DEC_MAX_REP, TL_ERR_INVALID,
               "%s: GQA group %d/%d unsupported (max %d)", what, n_h, n_kv, DEC_MAX_REP);
    TL_REQUIRE(kv_len_dev != nullptr, TL_ERR_INVALID, "%s: kv_len_dev is null", what);
    TL_REQUIRE(ws_bytes >= tl_attn_decode_ws(B, n_h, d, T_max), TL_ERR_WORKSPACE,
               "%s: workspace %zu < %zu", what, ws_bytes, tl_attn_decode_ws(B, n_h, d, T_max));
    if (B == 0) return TL_OK;
    const int n_splits = (T_max + DEC_CHUNK - 1) / DEC_CHUNK;
    const float sl2 = scale * 1.4426950408889634f;
    const dim3 g1(n_splits, n_kv, B), g2(n_h, B);
    // split phase on tensor cores (attn_decode_mma_kernel) unless TL_DECODE_ATTN=simt asks for the CUDA-core kernel
    const char* impl = getenv("TL_DECODE_ATTN");
    if (!(impl && impl[0] == 's')) {
        const int ns_m = (T_max + DEC_CHUNK_MMA - 1) / DEC_CHUNK_MMA;
        const dim3 gm(ns_m, n_kv, B);
        const size_t smem = (size_t)(16 + 4 * FA_BKV) * (d + 8) * sizeof(bf16);
#define TL_DEC_MMA(D_, ROWS_)                                                                                               \
        do {                                                                                                                \
            static bool done = false;                                                                                       \
            if (!done) { cudaFuncSetAttribute(attn_decode_mma_kernel<D_, ROWS_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); done = true; } \
            attn_decode_mma_kernel<D_, ROWS_><<<gm, FA_THREADS, smem, st>>>((const bf16*)q, (const bf16*)k_cache, (const bf16*)v_cache, \
                                                                             (float*)workspace, kv_len_dev, n_h, n_kv, T_max, ns_m, sl2, kv_start); \
            attn_decode_reduce_kernel<D_, ROWS_><<<g2, D_, 0, st>>>((const float*)workspace, (bf16*)out, kv_len_dev, n_h, n_kv, ns_m, \
                                                                     DEC_CHUNK_MMA, kv_start);                             \
        } while (0)
        if (kv_start) {
            if (d == 64) TL_DEC_MMA(64, true); else TL_DEC_MMA(128, true);
        } else {
            if (d == 64) TL_DEC_MMA(64, false); else TL_DEC_MMA(128, false);
        }
#undef TL_DEC_MMA
        return check_launch(what);
    }
#define TL_DEC_SIMT(D_, ROWS_)                                                                                              \
    do {                                                                                                                    \
        attn_decode_split_kernel<D_, ROWS_><<<g1, DEC_THREADS, 0, st>>>((const bf16*)q, (const bf16*)k_cache, (const bf16*)v_cache, \
                                                                         (float*)workspace, kv_len_dev, n_h, n_kv, T_max, n_splits, sl2, kv_start); \
        attn_decode_reduce_kernel<D_, ROWS_><<<g2, D_, 0, st>>>((const float*)workspace, (bf16*)out, kv_len_dev, n_h, n_kv, n_splits, \
                                                                 DEC_CHUNK, kv_start);                                     \
    } while (0)
    if (kv_start) {
        if (d == 64) TL_DEC_SIMT(64, true); else TL_DEC_SIMT(128, true);
    } else {
        if (d == 64) TL_DEC_SIMT(64, false); else TL_DEC_SIMT(128, false);
    }
#undef TL_DEC_SIMT
    return check_launch(what);
}
}  // namespace tl

// ================================================================================================ fused decode
// RoPE (+ Qwen3 q/k-norm) + KV-cache append + single-pass attention for ONE new token per batch row, short
// contexts (T_max <= FD_MAX_T).  One CTA per (query head, batch row): the rotated key/value of the new token are
// recomputed by every head of a GQA group (d multiply-adds) so no CTA has to wait for the cache write of another.
// Replaces three launches per layer (rope_kv_fwd, attn_decode_split, attn_decode_reduce) at decode time.
namespace tl {

constexpr int FD_THREADS = 128, FD_MAX_T = 2048;

// ROWS: row b is left-padded by kv_start[b] slots: the new token is rotated at position pos - kv_start[b] (it is still
// written to slot pos) and attends to keys kv_start[b]..pos only
template <int D, bool ROWS>
__global__ void __launch_bounds__(FD_THREADS) attn_decode_fused_kernel(
    const bf16* __restrict__ qkv, bf16* __restrict__ k_cache, bf16* __restrict__ v_cache, bf16* __restrict__ out,
    const int32_t* __restrict__ pos_dev, const bf16* __restrict__ cos_tab, const bf16* __restrict__ sin_tab,
    const bf16* __restrict__ q_norm_w, const bf16* __restrict__ k_norm_w, float eps, int n_h, int n_kv, int T_max,
    float scale_log2, const int32_t* __restrict__ kv_start) {
    constexpr int HALF = D / 2;
    // programmatic dependent launch: this grid may become resident while the qkv Linear is still running; wait for its
    // output here, and let the o-proj Linear behind us start prefetching its weights right away
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;");
    const int h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n_rep = n_h / n_kv, kvh = h / n_rep;
    const int pos = *pos_dev;                       // keys 0..pos-1 are cached; the new token is key `pos`
    int k_start = 0;                                // ROWS: first key this row attends to; the rotary position is
    if constexpr (ROWS) {                           // pos - k_start (the tables are read from k_start rows earlier)
        k_start = kv_start[b];
        cos_tab -= (size_t)k_start * HALF;
        sin_tab -= (size_t)k_start * HALF;
    }
    const int heads = n_h + 2 * n_kv;
    __shared__ __align__(16) float sq[D], sk[D], sv[D];
    __shared__ float sscore[FD_MAX_T + 1];
    __shared__ float sred[FD_THREADS / 32];
    __shared__ float s_bc[2];
    __shared__ __align__(16) float so[FD_THREADS / 32][D];

    // ---- RoPE of q (head h), k and v of the new token (kv head kvh); identical rounding to rope_kv_fwd_kernel
    const bf16* row = qkv + (size_t)b * heads * D;
    float q1 = 0.f, q2 = 0.f, k1 = 0.f, k2 = 0.f;
    if (tid < HALF) {
        q1 = bf2f(row[(size_t)h * D + tid]);
        q2 = bf2f(row[(size_t)h * D + tid + HALF]);
        k1 = bf2f(row[(size_t)(n_h + kvh) * D + tid]);
        k2 = bf2f(row[(size_t)(n_h + kvh) * D + tid + HALF]);
        sv[tid] = bf2f(row[(size_t)(n_h + n_kv + kvh) * D + tid]);
        sv[tid + HALF] = bf2f(row[(size_t)(n_h + n_kv + kvh) * D + tid + HALF]);
    }
    if (q_norm_w) {        // Qwen3: RMSNorm over the head dim (block reduction over the HALF active threads)
        float a = warp_sum(q1 * q1 + q2 * q2), c = warp_sum(k1 * k1 + k2 * k2);
        __shared__ float nr[2][FD_THREADS / 32];
        if (lane == 0) { nr[0][warp] = a; nr[1][warp] = c; }
        __syncthreads();
        a = c = 0.f;
#pragma unroll
        for (int w = 0; w < FD_THREADS / 32; ++w) { a += nr[0][w]; c += nr[1][w]; }
        const float rq = 1.0f / sqrtf(a / (float)D + eps), rk = 1.0f / sqrtf(c / (float)D + eps);
        if (tid < HALF) {
            q1 = rbf(bf2f(q_norm_w[tid]) * rbf(q1 * rq));
            q2 = rbf(bf2f(q_norm_w[tid + HALF]) * rbf(q2 * rq));
            k1 = rbf(bf2f(k_norm_w[tid]) * rbf(k1 * rk));
            k2 = rbf(bf2f(k_norm_w[tid + HALF]) * rbf(k2 * rk));
        }
    }
    if (tid < HALF) {
        const float c = bf2f(cos_tab[(size_t)pos * HALF + tid]), s = bf2f(sin_tab[(size_t)pos * HALF + tid]);
        sq[tid] = rbf(rbf(q1 * c) + rbf(-q2 * s));
        sq[tid + HALF] = rbf(rbf(q2 * c) + rbf(q1 * s));
        sk[tid] = rbf(rbf(k1 * c) + rbf(-k2 * s));
        sk[tid + HALF] = rbf(rbf(k2 * c) + rbf(k1 * s));
    }
    __syncthreads();
    if (h % n_rep == 0 && tid < D) {       // one head of the group appends the new key/value to the cache
        const size_t off = (((size_t)b * n_kv + kvh) * T_max + pos) * D + tid;
        k_cache[off] = f2bf(sk[tid]);
        v_cache[off] = f2bf(sv[tid]);
    }
    // ---- scores: one cached key per thread per round; the new key by warp 0
    const bf16* kb = k_cache + ((size_t)b * n_kv + kvh) * T_max * D;
    const bf16* vb = v_cache + ((size_t)b * n_kv + kvh) * T_max * D;
    float mx = -INFINITY;
    for (int key = tid; key < pos; key += FD_THREADS) {
        if constexpr (ROWS) if (key < k_start) continue;
        const uint4* kr = reinterpret_cast<const uint4*>(kb + (size_t)key * D);
        float acc = 0.f;
#pragma unroll 4
        for (int c = 0; c < D / 8; ++c) {
            const uint4 kv4 = kr[c];
            const uint32_t* k32 = reinterpret_cast<const uint32_t*>(&kv4);
            const float4 qa = *reinterpret_cast<const float4*>(&sq[c * 8]);
            const float4 qb = *reinterpret_cast<const float4*>(&sq[c * 8 + 4]);
            acc += bf16_lo(k32[0]) * qa.x + bf16_hi(k32[0]) * qa.y + bf16_lo(k32[1]) * qa.z + bf16_hi(k32[1]) * qa.w +
                   bf16_lo(k32[2]) * qb.x + bf16_hi(k32[2]) * qb.y + bf16_lo(k32[3]) * qb.z + bf16_hi(k32[3]) * qb.w;
        }
        acc *= scale_log2;
        sscore[key] = acc;
        mx = fmaxf(mx, acc);
    }
    if (warp == 0) {
        float acc = 0.f;
        for (int i = lane; i < D; i += 32) acc += sq[i] * sk[i];
        acc = warp_sum(acc) * scale_log2;
        if (lane == 0) sscore[pos] = acc;
        mx = fmaxf(mx, acc);
    }
    mx = warp_max(mx);
    if (lane == 0) sred[warp] = mx;
    __syncthreads();
    if (tid == 0) {
        float m = sred[0];
#pragma unroll
        for (int w = 1; w < FD_THREADS / 32; ++w) m = fmaxf(m, sred[w]);
        s_bc[0] = m;
    }
    __syncthreads();
    const float m_all = s_bc[0];
    float lsum = 0.f;
    for (int key = tid; key <= pos; key += FD_THREADS) {
        if constexpr (ROWS) if (key < k_start) continue;
        const float p = exp2f(sscore[key] - m_all);
        lsum += p;
        sscore[key] = rbf(p);           // P is cast to bf16 before P·V (SDPA contract); l uses the fp32 value
    }
    lsum = warp_sum(lsum);
    __syncthreads();
    if (lane == 0) sred[warp] = lsum;
    __syncthreads();
    // ---- P·V: threads own 8 output dims; key groups stride the cached keys
    constexpr int TPR = D / 8, KG = FD_THREADS / TPR;
    const int dd0 = (tid % TPR) * 8, kgi = tid / TPR;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    for (int key = kgi; key < pos; key += KG) {
        if constexpr (ROWS) if (key < k_start) continue;
        const uint4 vv = *reinterpret_cast<const uint4*>(vb + (size_t)key * D + dd0);
        const uint32_t* v32 = reinterpret_cast<const uint32_t*>(&vv);
        const float p = sscore[key];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            acc[2 * j] = fmaf(p, bf16_lo(v32[j]), acc[2 * j]);
            acc[2 * j + 1] = fmaf(p, bf16_hi(v32[j]), acc[2 * j + 1]);
        }
    }
    if (kgi == 0) {                      // the new token's value
        const float p = sscore[pos];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = fmaf(p, sv[dd0 + j], acc[j]);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        float v = acc[j];
#pragma unroll
        for (int off = TPR; off < 32; off <<= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
        acc[j] = v;
    }
    if (lane < TPR) {
#pragma unroll
        for (int j = 0; j < 8; ++j) so[warp][dd0 + j] = acc[j];
    }
    __syncthreads();
    if (tid < D) {
        float l = 0.f, o = 0.f;
#pragma unroll
        for (int w = 0; w < FD_THREADS / 32; ++w) { l += sred[w]; o += so[w][tid]; }
        out[((size_t)b * n_h + h) * D + tid] = f2bf(o / l);
    }
}

}  // namespace tl

namespace tl {
// launch configuration of the fused decode kernel; programmatic dependent launch is opt-in (see below)
static int attn_decode_fused_cfg(cudaLaunchConfig_t* cfg, cudaLaunchAttribute* attr, int d, int n_h, int n_kv, int T_max,
                                 const int32_t* pos_dev, int B, void* stream, const char* what) {
    TL_REQUIRE(d == 64 || d == 128, TL_ERR_INVALID, "%s: head_dim %d not in {64,128}", what, d);
    TL_REQUIRE(n_kv > 0 && n_h % n_kv == 0, TL_ERR_INVALID, "%s: n_h %% n_kv != 0", what);
    TL_REQUIRE(T_max <= FD_MAX_T, TL_ERR_INVALID, "%s: T_max %d > %d (use the split-KV path)", what, T_max, FD_MAX_T);
    TL_REQUIRE(pos_dev != nullptr, TL_ERR_INVALID, "%s: pos_dev is null", what);
    *cfg = {};
    cfg->gridDim = dim3(n_h, B);
    cfg->blockDim = dim3(FD_THREADS);
    cfg->dynamicSmemBytes = 0;
    cfg->stream = (cudaStream_t)stream;
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    static int use_pdl = -1;
    if (use_pdl < 0) {
        const char* e = getenv("TL_PDL");
        const char* e2 = getenv("TL_PDL_ATTN");
        // an early-resident attention grid competes with the Linear it overlaps for SMs, so the attribute is opt-in here (TL_PDL_ATTN=1); the weight-streaming Linears keep it on by default
        use_pdl = (!(e && e[0] == '0') && (e2 && e2[0] == '1')) ? 1 : 0;
    }
    cfg->attrs = attr;
    cfg->numAttrs = use_pdl ? 1 : 0;
    return TL_OK;
}
}  // namespace tl

extern "C" int tl_attn_decode_fused(const void* qkv, void* k_cache, void* v_cache, void* out, const int32_t* pos_dev,
                                    const void* cos_tab, const void* sin_tab, const void* q_norm_w, const void* k_norm_w,
                                    float eps, int B, int n_h, int n_kv, int d, int T_max, float scale, void* stream) {
    using namespace tl;
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute attr[1];
    const int rc = attn_decode_fused_cfg(&cfg, attr, d, n_h, n_kv, T_max, pos_dev, B, stream, "tl_attn_decode_fused");
    if (rc != TL_OK || B == 0) return rc;
    const float sl2 = scale * 1.4426950408889634f;
    if (d == 64)
        cudaLaunchKernelEx(&cfg, attn_decode_fused_kernel<64, false>, (const bf16*)qkv, (bf16*)k_cache, (bf16*)v_cache, (bf16*)out,
                           pos_dev, (const bf16*)cos_tab, (const bf16*)sin_tab, (const bf16*)q_norm_w, (const bf16*)k_norm_w, eps,
                           n_h, n_kv, T_max, sl2, (const int32_t*)nullptr);
    else
        cudaLaunchKernelEx(&cfg, attn_decode_fused_kernel<128, false>, (const bf16*)qkv, (bf16*)k_cache, (bf16*)v_cache, (bf16*)out,
                           pos_dev, (const bf16*)cos_tab, (const bf16*)sin_tab, (const bf16*)q_norm_w, (const bf16*)k_norm_w, eps,
                           n_h, n_kv, T_max, sl2, (const int32_t*)nullptr);
    return check_launch("tl_attn_decode_fused");
}

extern "C" int tl_attn_decode_fused_rows(const void* qkv, void* k_cache, void* v_cache, void* out, const int32_t* pos_dev,
                                         const void* cos_tab, const void* sin_tab, const void* q_norm_w, const void* k_norm_w,
                                         float eps, int B, int n_h, int n_kv, int d, int T_max, float scale,
                                         const int32_t* kv_start_dev, void* stream) {
    using namespace tl;
    TL_REQUIRE(kv_start_dev != nullptr, TL_ERR_INVALID, "tl_attn_decode_fused_rows: kv_start_dev is null");
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute attr[1];
    const int rc = attn_decode_fused_cfg(&cfg, attr, d, n_h, n_kv, T_max, pos_dev, B, stream, "tl_attn_decode_fused_rows");
    if (rc != TL_OK || B == 0) return rc;
    const float sl2 = scale * 1.4426950408889634f;
    if (d == 64)
        cudaLaunchKernelEx(&cfg, attn_decode_fused_kernel<64, true>, (const bf16*)qkv, (bf16*)k_cache, (bf16*)v_cache, (bf16*)out,
                           pos_dev, (const bf16*)cos_tab, (const bf16*)sin_tab, (const bf16*)q_norm_w, (const bf16*)k_norm_w, eps,
                           n_h, n_kv, T_max, sl2, kv_start_dev);
    else
        cudaLaunchKernelEx(&cfg, attn_decode_fused_kernel<128, true>, (const bf16*)qkv, (bf16*)k_cache, (bf16*)v_cache, (bf16*)out,
                           pos_dev, (const bf16*)cos_tab, (const bf16*)sin_tab, (const bf16*)q_norm_w, (const bf16*)k_norm_w, eps,
                           n_h, n_kv, T_max, sl2, kv_start_dev);
    return check_launch("tl_attn_decode_fused_rows");
}
