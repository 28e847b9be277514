// HBM-bound row kernels: RMSNorm, embedding gather, rotary tables, RoPE + KV-cache append.
// Rounding points follow the HF bf16 pipeline the reference executes (see include/tensorlink_b200.h).
#include "common.cuh"

namespace tl {

// ------------------------------------------------------------------------------------------------ RMSNorm
// one CTA per row, 16-byte vector loads kept in registers between the reduce and the scale pass
constexpr int NORM_THREADS = 128;
constexpr int NORM_MAXV = 8;   // H <= 128 * 8 * 8 = 8192

__global__ void __launch_bounds__(NORM_THREADS) rmsnorm_fwd_kernel(const bf16* __restrict__ x,
                                                                     const bf16* __restrict__ w,
                                                                     bf16* __restrict__ y,
                                                                     float* __restrict__ rstd_out, int H, float eps) {
    const int row = blockIdx.x;
    const int nvec = H >> 3;
    const uint4* xr = reinterpret_cast<const uint4*>(x + (size_t)row * H);
    uint4 v[NORM_MAXV];
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < NORM_MAXV; ++i) {
        int idx = threadIdx.x + i * NORM_THREADS;
        if (idx < nvec) {
            v[i] = xr[idx];
            const uint32_t* u = reinterpret_cast<const uint32_t*>(&v[i]);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                float a = bf16_lo(u[j]), b = bf16_hi(u[j]);
                ss += a * a + b * b;
            }
        }
    }
    __shared__ float red[NORM_THREADS / 32];
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int i = 0; i < NORM_THREADS / 32; ++i) tot += red[i];
    const float rstd = 1.0f / sqrtf(tot / (float)H + eps);
    if (rstd_out && threadIdx.x == 0) rstd_out[row] = rstd;
    const uint4* wr = reinterpret_cast<const uint4*>(w);
    uint4* yr = reinterpret_cast<uint4*>(y + (size_t)row * H);
#pragma unroll
    for (int i = 0; i < NORM_MAXV; ++i) {
        int idx = threadIdx.x + i * NORM_THREADS;
        if (idx < nvec) {
            uint4 wv = wr[idx], o;
            const uint32_t* u = reinterpret_cast<const uint32_t*>(&v[i]);
            const uint32_t* g = reinterpret_cast<const uint32_t*>(&wv);
            uint32_t* ou = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                float a = rbf(bf16_lo(u[j]) * rstd), b = rbf(bf16_hi(u[j]) * rstd);
                ou[j] = pack_bf16(bf16_lo(g[j]) * a, bf16_hi(g[j]) * b);
            }
            yr[idx] = o;
        }
    }
}

// ------------------------------------------------------------------------------------------------ embedding
__global__ void embed_fwd_kernel(const int64_t* __restrict__ ids, const bf16* __restrict__ table,
                                 bf16* __restrict__ out, int n_tokens, int H, int vocab) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= n_tokens) return;
    long long id = ids[warp];
    if (id < 0 || id >= vocab) id = 0;   // torch would raise; callers validate ids on the host
    const uint4* src = reinterpret_cast<const uint4*>(table + (size_t)id * H);
    uint4* dst = reinterpret_cast<uint4*>(out + (size_t)warp * H);
    for (int i = lane; i < (H >> 3); i += 32) dst[i] = src[i];
}

// ------------------------------------------------------------------------------------------------ rotary tables
__global__ void rope_table_kernel(const float* __restrict__ inv_freq, bf16* __restrict__ cos_tab,
                                  bf16* __restrict__ sin_tab, int max_pos, int half) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= max_pos * half) return;
    const int pos = idx / half, i = idx - pos * half;
    const float ang = (float)pos * inv_freq[i];
    cos_tab[idx] = f2bf(cosf(ang));
    sin_tab[idx] = f2bf(sinf(ang));
}

// ------------------------------------------------------------------------------------------------ RoPE + KV append
// one warp per (token, head) vector; lanes own pairs (i, i + d/2)
// ROWS: row b's token at cache slot t sits at rotary position t - kv_start[b] (left-padded rows); the pad slots below
// kv_start get a negative position and are rotated at position 0 instead (finite, never attended)
template <int D, bool ROWS>
__global__ void __launch_bounds__(128) rope_kv_fwd_kernel(const bf16* __restrict__ qkv, bf16* __restrict__ q_out,
                                                           bf16* __restrict__ k_cache, bf16* __restrict__ v_cache,
                                                           const int32_t* __restrict__ pos0_dev,
                                                           const bf16* __restrict__ cos_tab,
                                                           const bf16* __restrict__ sin_tab,
                                                           const bf16* __restrict__ q_norm_w,
                                                           const bf16* __restrict__ k_norm_w, float eps, int n_tokens,
                                                           int S, int n_h, int n_kv, int T_max,
                                                           const int32_t* __restrict__ kv_start) {
    constexpr int HALF = D / 2;
    constexpr int PAIRS = HALF / 32;   // pairs per lane: 1 (d=64) or 2 (d=128)
    const int heads = n_h + 2 * n_kv;
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (gw >= n_tokens * heads) return;
    const int n = gw / heads, h = gw - n * heads;
    const int b = n / S;
    const int pos = (pos0_dev ? *pos0_dev : 0) + (n - b * S);
    int rpos = pos;                                          // rotary position (the cache slot is always `pos`)
    if constexpr (ROWS) rpos = max(pos - kv_start[b], 0);
    const bf16* src = qkv + (size_t)n * heads * D + (size_t)h * D;
    float x1[PAIRS], x2[PAIRS];
#pragma unroll
    for (int p = 0; p < PAIRS; ++p) {
        x1[p] = bf2f(src[lane + 32 * p]);
        x2[p] = bf2f(src[lane + 32 * p + HALF]);
    }
    const bool is_q = h < n_h, is_k = !is_q && h < n_h + n_kv;
    if (!is_q && !is_k) {   // V: plain copy into the cache
        bf16* dst = v_cache + (((size_t)b * n_kv + (h - n_h - n_kv)) * T_max + pos) * D;
#pragma unroll
        for (int p = 0; p < PAIRS; ++p) {
            dst[lane + 32 * p] = f2bf(x1[p]);
            dst[lane + 32 * p + HALF] = f2bf(x2[p]);
        }
        return;
    }
    const bf16* nw = is_q ? q_norm_w : k_norm_w;
    if (nw) {   // Qwen3: RMSNorm over the head dim before RoPE
        float ss = 0.f;
#pragma unroll
        for (int p = 0; p < PAIRS; ++p) ss += x1[p] * x1[p] + x2[p] * x2[p];
        ss = warp_sum(ss);
        const float rstd = 1.0f / sqrtf(ss / (float)D + eps);
#pragma unroll
        for (int p = 0; p < PAIRS; ++p) {
            x1[p] = rbf(bf2f(nw[lane + 32 * p]) * rbf(x1[p] * rstd));
            x2[p] = rbf(bf2f(nw[lane + 32 * p + HALF]) * rbf(x2[p] * rstd));
        }
    }
    bf16* dst = is_q ? q_out + (size_t)n * n_h * D + (size_t)h * D
                     : k_cache + (((size_t)b * n_kv + (h - n_h)) * T_max + pos) * D;
#pragma unroll
    for (int p = 0; p < PAIRS; ++p) {
        const int i = lane + 32 * p;
        const float c = bf2f(cos_tab[(size_t)rpos * HALF + i]);
        const float s = bf2f(sin_tab[(size_t)rpos * HALF + i]);
        // (q * cos) + (rotate_half(q) * sin), every product and the sum rounded to bf16 like torch
        dst[i] = f2bf(rbf(x1[p] * c) + rbf(-x2[p] * s));
        dst[i + HALF] = f2bf(rbf(x2[p] * c) + rbf(x1[p] * s));
    }
}

}  // namespace tl

extern "C" {

int tl_rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd_out, int rows, int H, float eps, void* stream) {
    using namespace tl;
    TL_REQUIRE(rows >= 0 && H > 0 && H % 8 == 0 && H <= NORM_THREADS * NORM_MAXV * 8, TL_ERR_INVALID,
               "tl_rmsnorm_fwd: H=%d must be a multiple of 8 and <= %d", H, NORM_THREADS * NORM_MAXV * 8);
    if (rows == 0) return TL_OK;
    rmsnorm_fwd_kernel<<<rows, NORM_THREADS, 0, (cudaStream_t)stream>>>((const bf16*)x, (const bf16*)w, (bf16*)y,
                                                                        rstd_out, H, eps);
    return check_launch("tl_rmsnorm_fwd");
}

int tl_embed_fwd(const int64_t* ids, const void* table, void* out, int n_tokens, int H, int vocab, void* stream) {
    using namespace tl;
    TL_REQUIRE(H % 8 == 0 && n_tokens >= 0, TL_ERR_INVALID, "tl_embed_fwd: H=%d must be a multiple of 8", H);
    if (n_tokens == 0) return TL_OK;
    const int warps_per_block = 8;
    embed_fwd_kernel<<<(n_tokens + warps_per_block - 1) / warps_per_block, warps_per_block * 32, 0,
                       (cudaStream_t)stream>>>(ids, (const bf16*)table, (bf16*)out, n_tokens, H, vocab);
    return check_launch("tl_embed_fwd");
}

int tl_rope_table(const float* inv_freq, void* cos_tab, void* sin_tab, int max_pos, int half_dim, void* stream) {
    using namespace tl;
    TL_REQUIRE(max_pos > 0 && half_dim > 0, TL_ERR_INVALID, "tl_rope_table: bad shape");
    const int n = max_pos * half_dim;
    rope_table_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(inv_freq, (bf16*)cos_tab, (bf16*)sin_tab,
                                                                          max_pos, half_dim);
    return check_launch("tl_rope_table");
}

static int rope_kv_launch(const void* qkv, void* q_out, void* k_cache, void* v_cache, const int32_t* pos0_dev,
                          const void* cos_tab, const void* sin_tab, const void* q_norm_w, const void* k_norm_w, float eps,
                          int n_tokens, int S, int n_h, int n_kv, int d, int T_max, const int32_t* kv_start, void* stream,
                          const char* what) {
    using namespace tl;
    TL_REQUIRE(d == 64 || d == 128, TL_ERR_INVALID, "%s: head_dim %d not in {64,128}", what, d);
    TL_REQUIRE(S > 0 && n_tokens % S == 0, TL_ERR_INVALID, "%s: n_tokens %d not a multiple of S %d", what, n_tokens, S);
    if (n_tokens == 0) return TL_OK;
    const long long warps = (long long)n_tokens * (n_h + 2 * n_kv);
    const int grid = (int)((warps + 3) / 4);
    cudaStream_t st = (cudaStream_t)stream;
#define TL_ROPE_LAUNCH(D_, ROWS_)                                                                                          \
    rope_kv_fwd_kernel<D_, ROWS_><<<grid, 128, 0, st>>>((const bf16*)qkv, (bf16*)q_out, (bf16*)k_cache, (bf16*)v_cache,   \
                                                        pos0_dev, (const bf16*)cos_tab, (const bf16*)sin_tab,              \
                                                        (const bf16*)q_norm_w, (const bf16*)k_norm_w, eps, n_tokens, S,   \
                                                        n_h, n_kv, T_max, kv_start)
    if (kv_start) {
        if (d == 64) TL_ROPE_LAUNCH(64, true); else TL_ROPE_LAUNCH(128, true);
    } else {
        if (d == 64) TL_ROPE_LAUNCH(64, false); else TL_ROPE_LAUNCH(128, false);
    }
#undef TL_ROPE_LAUNCH
    return check_launch(what);
}

int tl_rope_kv_fwd(const void* qkv, void* q_out, void* k_cache, void* v_cache, const int32_t* pos0_dev,
                   const void* cos_tab, const void* sin_tab, const void* q_norm_w, const void* k_norm_w, float eps,
                   int n_tokens, int S, int n_h, int n_kv, int d, int T_max, void* stream) {
    return rope_kv_launch(qkv, q_out, k_cache, v_cache, pos0_dev, cos_tab, sin_tab, q_norm_w, k_norm_w, eps, n_tokens, S,
                          n_h, n_kv, d, T_max, nullptr, stream, "tl_rope_kv_fwd");
}

int tl_rope_kv_fwd_rows(const void* qkv, void* q_out, void* k_cache, void* v_cache, const int32_t* pos0_dev,
                        const void* cos_tab, const void* sin_tab, const void* q_norm_w, const void* k_norm_w, float eps,
                        int n_tokens, int S, int n_h, int n_kv, int d, int T_max, const int32_t* kv_start_dev,
                        void* stream) {
    using namespace tl;
    TL_REQUIRE(kv_start_dev != nullptr, TL_ERR_INVALID, "tl_rope_kv_fwd_rows: kv_start_dev is null");
    return rope_kv_launch(qkv, q_out, k_cache, v_cache, pos0_dev, cos_tab, sin_tab, q_norm_w, k_norm_w, eps, n_tokens, S,
                          n_h, n_kv, d, T_max, kv_start_dev, stream, "tl_rope_kv_fwd_rows");
}

}  // extern "C"
