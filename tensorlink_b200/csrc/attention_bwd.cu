// Causal GQA attention backward (training): recompute P from the saved log-sum-exp, two passes without atomics.
//   pass 0  D[b,h,s]   = sum_d dO * O                                   (fp32)
//   pass 1  dQ tile    = sum_kv  dS · K          dS = P ∘ (dO·V^T − D) · scale      (parallel over query tiles)
//   pass 2  dK,dV tile = sum_{q heads of the group, q tiles}  dS^T · Q ,  P^T · dO   (parallel over key tiles)
// Warp-level mma.sync kernels for sequences shorter than one 64-row tile; attention_wgmma.cu serves the rest.
// q/o/do/dq: [B,S,n_h,d] token-major;  k/v: [B,n_kv,T_max,d];  dk/dv: [B,n_h,T_max,d] (one partial per query head);
// lse/D: [B,n_h,S].
#include <stdlib.h>

#include "common.cuh"

namespace tl {

constexpr int AB_BQ = 64, AB_BKV = 64, AB_THREADS = 128;
constexpr float LOG2E = 1.4426950408889634f;

__device__ __forceinline__ void cp16(void* smem_dst, const void* gsrc, bool valid) {
    const uint32_t d = smem_u32(smem_dst);
    const int sz = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void ldsm4(uint32_t* r, const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldsm4t(uint32_t* r, const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void mma16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// ------------------------------------------------------------------------------------------------ pass 0
template <int D>
__global__ void attn_bwd_dot_kernel(const bf16* __restrict__ o, const bf16* __restrict__ dout, float* __restrict__ Dv, int S,
                                    int n_h, long long total) {
    const long long gw = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;   // one warp per (b, s, h)
    const int lane = threadIdx.x & 31;
    if (gw >= total) return;
    const long long bs = gw / n_h;
    const int h = (int)(gw - bs * n_h);
    const long long b = bs / S;
    const int s = (int)(bs - b * S);
    const bf16* po = o + (size_t)gw * D;
    const bf16* pd = dout + (size_t)gw * D;
    float acc = 0.f;
    for (int i = lane; i < D / 2; i += 32) {
        const uint32_t a = reinterpret_cast<const uint32_t*>(po)[i], c = reinterpret_cast<const uint32_t*>(pd)[i];
        acc += bf16_lo(a) * bf16_lo(c) + bf16_hi(a) * bf16_hi(c);
    }
    acc = warp_sum(acc);
    if (lane == 0) Dv[((size_t)b * n_h + h) * S + s] = acc;
}

// ------------------------------------------------------------------------------------------------ pass 1: dQ
// ROWS: keys below kv_start[b] are pad slots.  A query tile made only of pad rows writes dq = 0 and loads nothing; the
// KV loop starts at tile kv_start / 64, pad K/V rows load as zeros, and dS of pad keys (and so of pad query rows) is 0
// by select: pad q, dO, lse and D may hold anything.
template <int D, bool ROWS>
__global__ void __launch_bounds__(AB_THREADS) attn_bwd_dq_kernel(const bf16* __restrict__ q, const bf16* __restrict__ k_cache,
                                                                  const bf16* __restrict__ v_cache, const bf16* __restrict__ dout,
                                                                  const float* __restrict__ lse, const float* __restrict__ Dv,
                                                                  bf16* __restrict__ dq, int S, int n_h, int n_kv, int T_max,
                                                                  float scale, const int32_t* __restrict__ kv_start) {
    constexpr int LDS = D + 8, CPR = D / 8;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    bf16* sQ = reinterpret_cast<bf16*>(smem_raw);
    bf16* sdO = sQ + AB_BQ * LDS;
    bf16* sK = sdO + AB_BQ * LDS;            // [2][64][LDS]
    bf16* sV = sK + 2 * AB_BKV * LDS;        // [2][64][LDS]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
    const int qt = gridDim.x - 1 - blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int kvh = h / (n_h / n_kv), q0 = qt * AB_BQ;
    const bf16* qg = q + ((size_t)b * S) * n_h * D + (size_t)h * D;
    const bf16* dog = dout + ((size_t)b * S) * n_h * D + (size_t)h * D;
    const bf16* kg = k_cache + ((size_t)b * n_kv + kvh) * T_max * D;
    const bf16* vg = v_cache + ((size_t)b * n_kv + kvh) * T_max * D;
    int k_start = 0, t0 = 0;                               // first valid key and its tile
    if constexpr (ROWS) {
        k_start = kv_start[b];
        if (min(S, q0 + AB_BQ) <= k_start) {               // every query row of this tile is a pad row
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int row = q0 + warp * 16 + g + r * 8;
                if (row >= S) continue;
                bf16* dst = dq + ((size_t)b * S + row) * n_h * D + (size_t)h * D;
#pragma unroll
                for (int i = 0; i < D / 8; ++i) *reinterpret_cast<uint32_t*>(dst + i * 8 + 2 * t4) = 0u;
            }
            return;
        }
        t0 = k_start / AB_BKV;
    }
    for (int c = tid; c < AB_BQ * CPR; c += AB_THREADS) {
        const int r = c / CPR, cc = c - r * CPR;
        const bool ok = (q0 + r) < S;
        const size_t off = (size_t)(ok ? q0 + r : 0) * n_h * D + cc * 8;
        cp16(sQ + r * LDS + cc * 8, qg + off, ok);
        cp16(sdO + r * LDS + cc * 8, dog + off, ok);
    }
    auto load_kv = [&](int buf, int kv0) {
        for (int c = tid; c < AB_BKV * CPR; c += AB_THREADS) {
            const int r = c / CPR, cc = c - r * CPR;
            const bool ok = (kv0 + r) < S && (!ROWS || (kv0 + r) >= k_start);   // pad slots load as zeros
            const size_t off = (size_t)(ok ? kv0 + r : 0) * D + cc * 8;
            cp16(sK + (buf * AB_BKV + r) * LDS + cc * 8, kg + off, ok);
            cp16(sV + (buf * AB_BKV + r) * LDS + cc * 8, vg + off, ok);
        }
    };
    const int n_tiles = (min(S, q0 + AB_BQ) + AB_BKV - 1) / AB_BKV;
    load_kv(0, t0 * AB_BKV);
    cp_commit();
    float acc[D / 8][4];
#pragma unroll
    for (int i = 0; i < D / 8; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
    const int row0 = q0 + warp * 16 + g;
    float lse2[2], dvr[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = row0 + r * 8;
        const bool ok = row < S;
        lse2[r] = ok ? lse[((size_t)b * n_h + h) * S + row] * LOG2E : 0.f;
        dvr[r] = ok ? Dv[((size_t)b * n_h + h) * S + row] : 0.f;
    }
    const float sl2 = scale * LOG2E;
    for (int it = t0; it < n_tiles; ++it) {
        const int buf = (it - t0) & 1;
        if (it + 1 < n_tiles) load_kv(buf ^ 1, (it + 1) * AB_BKV);
        cp_commit();
        cp_wait<1>();
        __syncthreads();
        const bf16* sKb = sK + buf * AB_BKV * LDS;
        const bf16* sVb = sV + buf * AB_BKV * LDS;
        float s[AB_BKV / 8][4], dp[AB_BKV / 8][4];
#pragma unroll
        for (int i = 0; i < AB_BKV / 8; ++i) {
            s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
            dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f;
        }
#pragma unroll
        for (int ks = 0; ks < D / 16; ++ks) {
            uint32_t qa[4], da[4];
            ldsm4(qa, sQ + (warp * 16 + (lane & 15)) * LDS + ks * 16 + (lane >> 4) * 8);
            ldsm4(da, sdO + (warp * 16 + (lane & 15)) * LDS + ks * 16 + (lane >> 4) * 8);
#pragma unroll
            for (int np = 0; np < AB_BKV / 16; ++np) {
                uint32_t kb[4], vb[4];
                const int mi = lane >> 3;
                const int off = (np * 16 + (mi >> 1) * 8 + (lane & 7)) * LDS + ks * 16 + (mi & 1) * 8;
                ldsm4(kb, sKb + off);
                ldsm4(vb, sVb + off);
                mma16816(s[2 * np], qa, kb[0], kb[1]);
                mma16816(s[2 * np + 1], qa, kb[2], kb[3]);
                mma16816(dp[2 * np], da, vb[0], vb[1]);
                mma16816(dp[2 * np + 1], da, vb[2], vb[3]);
            }
        }
        const int kv0 = it * AB_BKV;
        uint32_t dsf[AB_BKV / 16][4];
#pragma unroll
        for (int i = 0; i < AB_BKV / 8; ++i) {
            float ds[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = kv0 + i * 8 + 2 * t4 + (e & 1);
                const int r = e >> 1;
                const int qpos = row0 + r * 8;
                if constexpr (ROWS) {       // key >= k_start also masks pad query rows (key <= qpos < k_start)
                    const bool ok = key <= qpos && key < S && key >= k_start;
                    ds[e] = ok ? exp2f(s[i][e] * sl2 - lse2[r]) * (dp[i][e] - dvr[r]) * scale : 0.f;
                } else {
                    const float p = (key > qpos || key >= S) ? 0.f : exp2f(s[i][e] * sl2 - lse2[r]);
                    ds[e] = p * (dp[i][e] - dvr[r]) * scale;
                }
            }
            dsf[i >> 1][(i & 1) * 2] = pack_bf16(ds[0], ds[1]);
            dsf[i >> 1][(i & 1) * 2 + 1] = pack_bf16(ds[2], ds[3]);
        }
#pragma unroll
        for (int kk = 0; kk < AB_BKV / 16; ++kk) {
#pragma unroll
            for (int dpi = 0; dpi < D / 16; ++dpi) {
                uint32_t kb[4];
                const int mi = lane >> 3;
                ldsm4t(kb, sKb + (kk * 16 + (mi & 1) * 8 + (lane & 7)) * LDS + dpi * 16 + (mi >> 1) * 8);
                mma16816(acc[2 * dpi], dsf[kk], kb[0], kb[1]);
                mma16816(acc[2 * dpi + 1], dsf[kk], kb[2], kb[3]);
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = row0 + r * 8;
        if (row >= S) continue;
        bf16* dst = dq + ((size_t)b * S + row) * n_h * D + (size_t)h * D;
#pragma unroll
        for (int i = 0; i < D / 8; ++i)
            *reinterpret_cast<uint32_t*>(dst + i * 8 + 2 * t4) = pack_bf16(acc[i][2 * r], acc[i][2 * r + 1]);
    }
}

// ------------------------------------------------------------------------------------------------ pass 2: dK, dV
// ROWS: a key tile lying wholly below kv_start[b] writes dk = dv = 0 and loads nothing.  Pad K/V rows and the Q / dO
// rows of pad queries load as zeros, and P / dS of pad keys and pad query rows are 0 by select, so pad key rows end as
// exact zeros.
template <int D, bool ROWS>
__global__ void __launch_bounds__(AB_THREADS) attn_bwd_dkv_kernel(const bf16* __restrict__ q, const bf16* __restrict__ k_cache,
                                                                   const bf16* __restrict__ v_cache, const bf16* __restrict__ dout,
                                                                   const float* __restrict__ lse, const float* __restrict__ Dv,
                                                                   bf16* __restrict__ dk, bf16* __restrict__ dv, int S, int n_h,
                                                                   int n_kv, int T_max, float scale,
                                                                   const int32_t* __restrict__ kv_start) {
    constexpr int LDS = D + 8, CPR = D / 8;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    bf16* sK = reinterpret_cast<bf16*>(smem_raw);      // [64][LDS]
    bf16* sV = sK + AB_BKV * LDS;
    bf16* sQ = sV + AB_BKV * LDS;                      // [2][64][LDS]
    bf16* sdO = sQ + 2 * AB_BQ * LDS;                  // [2][64][LDS]
    float* sL = reinterpret_cast<float*>(sdO + 2 * AB_BQ * LDS);   // [2][64]  lse * log2e
    float* sD = sL + 2 * AB_BQ;                                    // [2][64]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
    // one CTA per (key tile, QUERY head): dK/dV come out as one partial per query head, summed over the GQA group by
    // the RoPE backward kernel (7x more CTAs than looping the group inside one CTA, no atomics)
    const int kt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int n_rep = n_h / n_kv, kvh = h / n_rep, kv0 = kt * AB_BKV;
    const bf16* kg = k_cache + ((size_t)b * n_kv + kvh) * T_max * D;
    const bf16* vg = v_cache + ((size_t)b * n_kv + kvh) * T_max * D;
    int k_start = 0;
    if constexpr (ROWS) {
        k_start = kv_start[b];
        if (kv0 + AB_BKV <= k_start) {                     // every key of this tile is a pad slot
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int key = kv0 + warp * 16 + g + r * 8;
                if (key >= S) continue;
                bf16* dkd = dk + (((size_t)b * n_h + h) * T_max + key) * D;
                bf16* dvd = dv + (((size_t)b * n_h + h) * T_max + key) * D;
#pragma unroll
                for (int i = 0; i < D / 8; ++i) {
                    *reinterpret_cast<uint32_t*>(dkd + i * 8 + 2 * t4) = 0u;
                    *reinterpret_cast<uint32_t*>(dvd + i * 8 + 2 * t4) = 0u;
                }
            }
            return;
        }
    }
    for (int c = tid; c < AB_BKV * CPR; c += AB_THREADS) {
        const int r = c / CPR, cc = c - r * CPR;
        const bool ok = (kv0 + r) < S && (!ROWS || (kv0 + r) >= k_start);   // pad slots load as zeros
        const size_t off = (size_t)(ok ? kv0 + r : 0) * D + cc * 8;
        cp16(sK + r * LDS + cc * 8, kg + off, ok);
        cp16(sV + r * LDS + cc * 8, vg + off, ok);
    }
    const int qt_first = kv0 / AB_BQ, n_qt = (S + AB_BQ - 1) / AB_BQ;
    const int per_head = n_qt - qt_first;
    const int n_iter = per_head;
    auto load_q = [&](int buf, int iter) {
        const int qt = qt_first + iter;
        const int q0 = qt * AB_BQ;
        const bf16* qg = q + ((size_t)b * S) * n_h * D + (size_t)h * D;
        const bf16* dog = dout + ((size_t)b * S) * n_h * D + (size_t)h * D;
        for (int c = tid; c < AB_BQ * CPR; c += AB_THREADS) {
            const int r = c / CPR, cc = c - r * CPR;
            const bool ok = (q0 + r) < S && (!ROWS || (q0 + r) >= k_start);   // pad query rows load as zeros
            const size_t off = (size_t)(ok ? q0 + r : 0) * n_h * D + cc * 8;
            cp16(sQ + (buf * AB_BQ + r) * LDS + cc * 8, qg + off, ok);
            cp16(sdO + (buf * AB_BQ + r) * LDS + cc * 8, dog + off, ok);
        }
        if (tid < AB_BQ) {
            const bool ok = (q0 + tid) < S && (!ROWS || (q0 + tid) >= k_start);
            const size_t idx = ((size_t)b * n_h + h) * S + (ok ? q0 + tid : 0);
            sL[buf * AB_BQ + tid] = ok ? lse[idx] * LOG2E : INFINITY;   // +inf -> P = 0 for padded queries
            sD[buf * AB_BQ + tid] = ok ? Dv[idx] : 0.f;
        }
    };
    if (n_iter > 0) load_q(0, 0);
    cp_commit();
    float dka[D / 8][4], dva[D / 8][4];
#pragma unroll
    for (int i = 0; i < D / 8; ++i) {
        dka[i][0] = dka[i][1] = dka[i][2] = dka[i][3] = 0.f;
        dva[i][0] = dva[i][1] = dva[i][2] = dva[i][3] = 0.f;
    }
    const float sl2 = scale * LOG2E;
    const int key_row0 = kv0 + warp * 16 + g;
    for (int it = 0; it < n_iter; ++it) {
        const int buf = it & 1;
        if (it + 1 < n_iter) load_q(buf ^ 1, it + 1);
        cp_commit();
        cp_wait<1>();
        __syncthreads();
        const int qt = qt_first + it, q0 = qt * AB_BQ;
        const bf16* sQb = sQ + buf * AB_BQ * LDS;
        const bf16* sdOb = sdO + buf * AB_BQ * LDS;
        const float* sLb = sL + buf * AB_BQ;
        const float* sDb = sD + buf * AB_BQ;
#pragma unroll
        for (int half = 0; half < 2; ++half) {          // 32 query columns at a time (register pressure)
            float st[4][4], dpt[4][4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                st[i][0] = st[i][1] = st[i][2] = st[i][3] = 0.f;
                dpt[i][0] = dpt[i][1] = dpt[i][2] = dpt[i][3] = 0.f;
            }
#pragma unroll
            for (int ks = 0; ks < D / 16; ++ks) {
                uint32_t ka[4], va[4];
                ldsm4(ka, sK + (warp * 16 + (lane & 15)) * LDS + ks * 16 + (lane >> 4) * 8);
                ldsm4(va, sV + (warp * 16 + (lane & 15)) * LDS + ks * 16 + (lane >> 4) * 8);
#pragma unroll
                for (int np = 0; np < 2; ++np) {
                    uint32_t qb[4], ob[4];
                    const int mi = lane >> 3;
                    const int off = (half * 32 + np * 16 + (mi >> 1) * 8 + (lane & 7)) * LDS + ks * 16 + (mi & 1) * 8;
                    ldsm4(qb, sQb + off);
                    ldsm4(ob, sdOb + off);
                    mma16816(st[2 * np], ka, qb[0], qb[1]);
                    mma16816(st[2 * np + 1], ka, qb[2], qb[3]);
                    mma16816(dpt[2 * np], va, ob[0], ob[1]);
                    mma16816(dpt[2 * np + 1], va, ob[2], ob[3]);
                }
            }
            uint32_t pf[2][4], dsf[2][4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                float p[4], ds[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int qc = half * 32 + i * 8 + 2 * t4 + (e & 1);        // query column inside the tile
                    const int key = key_row0 + (e >> 1) * 8;
                    const int qpos = q0 + qc;
                    // ROWS: key >= k_start also masks pad query rows (key <= qpos < k_start); dS = P·(...) stays exact
                    // zero there, every operand of a pad row or slot having loaded as zero (D as 0)
                    p[e] = (key > qpos || key >= S || (ROWS && key < k_start)) ? 0.f : exp2f(st[i][e] * sl2 - sLb[qc]);
                    ds[e] = p[e] * (dpt[i][e] - sDb[qc]) * scale;
                }
                pf[i >> 1][(i & 1) * 2] = pack_bf16(p[0], p[1]);
                pf[i >> 1][(i & 1) * 2 + 1] = pack_bf16(p[2], p[3]);
                dsf[i >> 1][(i & 1) * 2] = pack_bf16(ds[0], ds[1]);
                dsf[i >> 1][(i & 1) * 2 + 1] = pack_bf16(ds[2], ds[3]);
            }
#pragma unroll
            for (int kk = 0; kk < 2; ++kk) {
#pragma unroll
                for (int dpi = 0; dpi < D / 16; ++dpi) {
                    uint32_t ob[4], qb[4];
                    const int mi = lane >> 3;
                    const int off = (half * 32 + kk * 16 + (mi & 1) * 8 + (lane & 7)) * LDS + dpi * 16 + (mi >> 1) * 8;
                    ldsm4t(ob, sdOb + off);
                    ldsm4t(qb, sQb + off);
                    mma16816(dva[2 * dpi], pf[kk], ob[0], ob[1]);
                    mma16816(dva[2 * dpi + 1], pf[kk], ob[2], ob[3]);
                    mma16816(dka[2 * dpi], dsf[kk], qb[0], qb[1]);
                    mma16816(dka[2 * dpi + 1], dsf[kk], qb[2], qb[3]);
                }
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int key = key_row0 + r * 8;
        if (key >= S) continue;
        bf16* dkd = dk + (((size_t)b * n_h + h) * T_max + key) * D;
        bf16* dvd = dv + (((size_t)b * n_h + h) * T_max + key) * D;
#pragma unroll
        for (int i = 0; i < D / 8; ++i) {
            *reinterpret_cast<uint32_t*>(dkd + i * 8 + 2 * t4) = pack_bf16(dka[i][2 * r], dka[i][2 * r + 1]);
            *reinterpret_cast<uint32_t*>(dvd + i * 8 + 2 * t4) = pack_bf16(dva[i][2 * r], dva[i][2 * r + 1]);
        }
    }
}

}  // namespace tl

namespace tl {
int attn_bwd_wgmma(const void* q, const void* k_cache, const void* v_cache, const void* dout, const float* lse, const float* Dv,
                   void* dq, void* dk, void* dv, int B, int S, int n_h, int n_kv, int d, int T_max, float scale,
                   const int32_t* kv_start, cudaStream_t st);

// kv_start (int32[B], device) non-null: the left-padded instantiations (ROWS)
static int attn_bwd_launch(const void* q, const void* k_cache, const void* v_cache, const void* out, const void* dout,
                           const float* lse, void* dq, void* dk, void* dv, void* workspace, size_t ws_bytes, int B, int S,
                           int n_h, int n_kv, int d, int T_max, float scale, const int32_t* kv_start, cudaStream_t st,
                           const char* what) {
    TL_REQUIRE(d == 64 || d == 128, TL_ERR_INVALID, "%s: head_dim %d not in {64,128}", what, d);
    TL_REQUIRE(n_kv > 0 && n_h % n_kv == 0 && S <= T_max, TL_ERR_INVALID, "%s: bad head/sequence configuration", what);
    TL_REQUIRE(ws_bytes >= tl_attn_bwd_ws(B, S, n_h), TL_ERR_WORKSPACE, "%s: workspace %zu < %zu", what, ws_bytes,
               tl_attn_bwd_ws(B, S, n_h));
    if (B == 0 || S == 0) return TL_OK;
    float* Dv = (float*)workspace;
    const long long total = (long long)B * S * n_h;
    const int g0 = (int)((total * 32 + 255) / 256);
    const dim3 g1((S + AB_BQ - 1) / AB_BQ, n_h, B), g2((S + AB_BKV - 1) / AB_BKV, n_h, B);
    {   // wgmma kernels (attention_wgmma.cu) from one full 64-row tile upwards; TL_ATTN_BWD=mma|wgmma forces a path
        const char* e = getenv("TL_ATTN_BWD");
        const int impl = !e ? 0 : (e[0] == 'm' ? 1 : (e[0] == 'w' ? 2 : 0));
        if (impl == 2 || (impl == 0 && S >= AB_BQ)) {
            if (d == 64) attn_bwd_dot_kernel<64><<<g0, 256, 0, st>>>((const bf16*)out, (const bf16*)dout, Dv, S, n_h, total);
            else attn_bwd_dot_kernel<128><<<g0, 256, 0, st>>>((const bf16*)out, (const bf16*)dout, Dv, S, n_h, total);
            return attn_bwd_wgmma(q, k_cache, v_cache, dout, lse, Dv, dq, dk, dv, B, S, n_h, n_kv, d, T_max, scale, kv_start, st);
        }
    }
    const size_t sm1 = (size_t)6 * 64 * (d + 8) * sizeof(bf16);
    const size_t sm2 = (size_t)6 * 64 * (d + 8) * sizeof(bf16) + 4 * 64 * sizeof(float);
#define TL_AB_BWD(D_, ROWS_)                                                                                                \
    do {                                                                                                                    \
        static bool done = false;                                                                                           \
        if (!done) {                                                                                                        \
            cudaFuncSetAttribute(attn_bwd_dq_kernel<D_, ROWS_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm1);      \
            cudaFuncSetAttribute(attn_bwd_dkv_kernel<D_, ROWS_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm2);     \
            done = true;                                                                                                    \
        }                                                                                                                   \
        attn_bwd_dot_kernel<D_><<<g0, 256, 0, st>>>((const bf16*)out, (const bf16*)dout, Dv, S, n_h, total);                \
        attn_bwd_dq_kernel<D_, ROWS_><<<g1, AB_THREADS, sm1, st>>>((const bf16*)q, (const bf16*)k_cache, (const bf16*)v_cache, \
                                                                   (const bf16*)dout, lse, Dv, (bf16*)dq, S, n_h, n_kv,     \
                                                                   T_max, scale, kv_start);                                 \
        attn_bwd_dkv_kernel<D_, ROWS_><<<g2, AB_THREADS, sm2, st>>>((const bf16*)q, (const bf16*)k_cache,                   \
                                                                    (const bf16*)v_cache, (const bf16*)dout, lse, Dv,       \
                                                                    (bf16*)dk, (bf16*)dv, S, n_h, n_kv, T_max, scale,       \
                                                                    kv_start);                                              \
    } while (0)
    if (kv_start) {
        if (d == 64) TL_AB_BWD(64, true); else TL_AB_BWD(128, true);
    } else {
        if (d == 64) TL_AB_BWD(64, false); else TL_AB_BWD(128, false);
    }
#undef TL_AB_BWD
    return check_launch(what);
}
}  // namespace tl

extern "C" {

size_t tl_attn_bwd_ws(int B, int S, int n_h) { return (size_t)B * n_h * S * sizeof(float); }

int tl_attn_bwd(const void* q, const void* k_cache, const void* v_cache, const void* out, const void* dout, const float* lse,
                void* dq, void* dk, void* dv, void* workspace, size_t ws_bytes, int B, int S, int n_h, int n_kv, int d,
                int T_max, float scale, void* stream) {
    return tl::attn_bwd_launch(q, k_cache, v_cache, out, dout, lse, dq, dk, dv, workspace, ws_bytes, B, S, n_h, n_kv, d,
                               T_max, scale, nullptr, (cudaStream_t)stream, "tl_attn_bwd");
}

int tl_attn_bwd_rows(const void* q, const void* k_cache, const void* v_cache, const void* out, const void* dout,
                     const float* lse, void* dq, void* dk, void* dv, void* workspace, size_t ws_bytes, int B, int S, int n_h,
                     int n_kv, int d, int T_max, float scale, const int32_t* kv_start_dev, void* stream) {
    using namespace tl;
    TL_REQUIRE(kv_start_dev != nullptr, TL_ERR_INVALID, "tl_attn_bwd_rows: kv_start_dev is null");
    return attn_bwd_launch(q, k_cache, v_cache, out, dout, lse, dq, dk, dv, workspace, ws_bytes, B, S, n_h, n_kv, d, T_max,
                           scale, kv_start_dev, (cudaStream_t)stream, "tl_attn_bwd_rows");
}

}  // extern "C"
