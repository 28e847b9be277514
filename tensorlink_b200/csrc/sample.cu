// Token sampling on the device: temperature -> top-k -> top-p -> multinomial draw, one CTA per row.
//
// The reference hands generation to HF ``generate`` (tensorlink/ml/module.py:763-769, ml/worker.py:403-404), whose
// sampling path is ``TemperatureLogitsWarper`` -> ``TopKLogitsWarper`` -> ``TopPLogitsWarper`` -> ``torch.multinomial``
// on the host's copy of the logits.  Here the logits never leave the last stage: this kernel reads the bf16 row the
// lm_head just wrote and stores one int64 id (into the first stage's mailbox on a multi-stage job).
//
// Everything is decided on a histogram over the 65536 possible bf16 bit patterns (integer atomics: deterministic):
//   * max                = highest occupied bin
//   * top-k threshold    = value of the k-th largest logit; every logit >= it is kept (HF: `scores < topk[-1]` removed)
//   * top-p threshold    = walking the bins downwards, a bin is kept while the probability mass ABOVE it is < top_p
//                          (HF removes ascending-cumulative-mass <= 1 - top_p and always keeps the top token); bf16
//                          logits tie often, and ties at the threshold are all kept
//   * draw               = Philox4x32-10(seed; row, counter) -> u in [0,1); inverse CDF over the kept tokens in index
//                          order (chunked prefix sums in a fixed order: a seed reproduces its tokens)
// The per-row counter lives in device memory and is advanced by the kernel, so a captured CUDA graph draws a fresh
// number on every replay.
#include "common.cuh"

namespace tl {

constexpr int SM_THREADS = 1024;
constexpr int SM_BINS = 65536;
constexpr int SM_PER = SM_BINS / SM_THREADS;      // bins per thread in the scans

__device__ __forceinline__ uint32_t bf16_key(uint16_t bits) {       // monotone: larger value -> larger key
    return (bits & 0x8000u) ? (uint32_t)(uint16_t)~bits : (uint32_t)(bits | 0x8000u);
}
__device__ __forceinline__ float key_value(uint32_t key) {
    const uint16_t bits = (key & 0x8000u) ? (uint16_t)(key & 0x7fffu) : (uint16_t)~key;
    return __uint_as_float(((uint32_t)bits) << 16);
}

__device__ __forceinline__ void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
    const uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
}
__device__ float philox_uniform(unsigned long long seed, uint32_t row, uint32_t counter) {
    uint32_t c[4] = {counter, row, 0x5eed5eedu, 0u};
    uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        philox_round(c, k0, k1);
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    return (float)(c[0] >> 8) * (1.0f / 16777216.0f);       // 24 random bits: [0, 1)
}

// exclusive block scan of one double per thread, in thread order (deterministic); returns the total through *total
__device__ double block_excl_scan(double v, double* s_warp, double* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
        double w = s_warp[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const double y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        s_warp[lane] = w;
    }
    __syncthreads();
    const double before = (warp ? s_warp[warp - 1] : 0.0) + (x - v);
    *total = s_warp[31];
    __syncthreads();
    return before;
}

// The row analysis of the rules above: the histogram of the row's bf16 keys in ``hist`` (this row's SM_BINS bins in
// global memory), then the max, the top-k key, the top-p key and the kept mass Z_kept of the bins.  Every kernel that
// samples from a warped bf16 row (sample_kernel, spec_rows_kernel) calls this one function, so they keep the same
// tokens with the same weights.  s_warp / s_sel / s_val: the CTA's shared scratch.
struct RowStats {
    float x_max;        // the max logit / temperature: weight(key) = __expf(key_value(key) * inv_temp - x_max)
    int p_key;          // kept: key >= p_key
    double Z_kept;      // the kept mass, summed over the bins
};

__device__ __forceinline__ RowStats row_analysis(const uint16_t* __restrict__ lr, int V, float inv_temp, int top_k, float top_p,
                                                 uint32_t* __restrict__ hist, double* s_warp, int* s_sel, double* s_val) {
    const int tid = threadIdx.x;
    for (int i = tid; i < SM_BINS; i += SM_THREADS) hist[i] = 0u;
    __syncthreads();
    for (int i = tid; i < V; i += SM_THREADS) atomicAdd(&hist[bf16_key(lr[i])], 1u);
    __syncthreads();
    // this thread owns bins [hi_key - SM_PER + 1, hi_key], walked downwards: thread 0 holds the largest values
    const int hi_key = SM_BINS - 1 - tid * SM_PER;
    uint32_t cnt[SM_PER];
    uint32_t local_n = 0;
#pragma unroll 8
    for (int j = 0; j < SM_PER; ++j) {
        cnt[j] = hist[hi_key - j];
        local_n += cnt[j];
    }
    // ---- max: the first occupied bin from the top
    double tot;
    const double n_before = block_excl_scan((double)local_n, s_warp, &tot);
    if (n_before == 0.0 && local_n > 0) {
        for (int j = 0; j < SM_PER; ++j)
            if (cnt[j]) { s_sel[0] = hi_key - j; break; }
    }
    __syncthreads();
    const int max_key = s_sel[0];
    const float x_max = key_value((uint32_t)max_key) * inv_temp;
    // ---- top-k: the bin holding the k-th largest logit (every logit of that bin is kept)
    int k_key = 0;                                   // keep everything by default
    if (top_k > 0 && top_k < V) {
        if (n_before < (double)top_k && n_before + (double)local_n >= (double)top_k) {
            double c = n_before;
            for (int j = 0; j < SM_PER; ++j) {
                c += (double)cnt[j];
                if (c >= (double)top_k) { s_sel[1] = hi_key - j; break; }
            }
        }
        __syncthreads();
        k_key = s_sel[1];
    }
    // ---- probability mass per thread over the bins that survive top-k (fixed order -> deterministic)
    double local_m = 0.0;
    for (int j = 0; j < SM_PER; ++j) {
        const int key = hi_key - j;
        if (cnt[j] && key >= k_key) local_m += (double)cnt[j] * (double)__expf(key_value((uint32_t)key) * inv_temp - x_max);
    }
    double Z;
    const double m_before = block_excl_scan(local_m, s_warp, &Z);
    // ---- top-p: keep a bin while the mass above it is < top_p * Z; the lowest kept bin is the threshold
    int p_key = k_key;
    double Z_kept = Z;
    if (top_p < 1.0f) {
        const double lim = (double)top_p * Z;
        if (tid == 0) { s_sel[2] = k_key; s_val[0] = Z; }
        __syncthreads();
        // the thread whose range contains the crossing point: mass before its range < lim <= mass through its range
        if (m_before < lim && m_before + local_m >= lim) {
            double c = m_before;
            for (int j = 0; j < SM_PER; ++j) {
                const int key = hi_key - j;
                if (!(cnt[j] && key >= k_key)) continue;
                const double w = (double)cnt[j] * (double)__expf(key_value((uint32_t)key) * inv_temp - x_max);
                if (c < lim) { s_sel[2] = key; s_val[0] = c + w; }     // kept: mass above it is still below the limit
                c += w;
            }
        }
        __syncthreads();
        p_key = s_sel[2];
        Z_kept = s_val[0];
    }
    return RowStats{x_max, p_key, Z_kept};
}

// LOG: once p_key is known, a pass over the row stores it into the score log (common.cuh LogDesc): the raw logit, and
// x / temperature on the kept set, -inf elsewhere.  The pass strides by the CTA's width, so its stores coalesce (the
// draw's per-thread ranges would scatter them).  The CTAs (rows) share the log column, so the last CTA out advances it.
// The draw itself does not depend on LOG.
template <bool LOG = false>
__global__ void __launch_bounds__(SM_THREADS) sample_kernel(const bf16* __restrict__ logits, int64_t* __restrict__ ids_out, int V,
                                                            float inv_temp, int top_k, float top_p, unsigned long long seed,
                                                            int32_t* __restrict__ counters, uint32_t* __restrict__ hist_all,
                                                            LogDesc lg) {
    const int row = blockIdx.x, tid = threadIdx.x;
    const uint16_t* lr = reinterpret_cast<const uint16_t*>(logits) + (size_t)row * V;
    __shared__ double s_warp[32];
    __shared__ int s_sel[4];
    __shared__ double s_val[2];
    const auto [x_max, p_key, Z_kept] = row_analysis(lr, V, inv_temp, top_k, top_p, hist_all + (size_t)row * SM_BINS, s_warp,
                                                     s_sel, s_val);
    // ---- draw and invert the CDF over the kept tokens in index order
    const uint32_t ctr = (uint32_t)counters[row];
    const double target = (double)philox_uniform(seed, (uint32_t)row, ctr) * Z_kept;
    const int per = (V + SM_THREADS - 1) / SM_THREADS;
    const int i0 = tid * per, i1 = min(V, i0 + per);
    float *raw = nullptr, *proc = nullptr;
    if (LOG && log_rows(lg, *lg.col, row, V, &raw, &proc)) {
        for (int i = tid; i < V; i += SM_THREADS) {          // interleaved, not the draw's per-thread ranges: coalesced stores
            const float x = __uint_as_float((uint32_t)lr[i] << 16);
            if (raw) raw[i] = x;
            if (proc) proc[i] = (int)bf16_key(lr[i]) >= p_key ? __fdiv_rn(x, lg.temperature) : -INFINITY;
        }
    }
    double local_w = 0.0;
    for (int i = i0; i < i1; ++i) {
        const uint32_t key = bf16_key(lr[i]);
        if ((int)key >= p_key) local_w += (double)__expf(key_value(key) * inv_temp - x_max);
    }
    double W;
    const double w_before = block_excl_scan(local_w, s_warp, &W);
    if (tid == 0) s_sel[3] = -1;
    __syncthreads();
    if (local_w > 0.0 && w_before <= target && target < w_before + local_w) {
        double c = w_before;
        int pick = -1;
        for (int i = i0; i < i1; ++i) {
            const uint32_t key = bf16_key(lr[i]);
            if ((int)key < p_key) continue;
            pick = i;
            c += (double)__expf(key_value(key) * inv_temp - x_max);
            if (target < c) break;
        }
        s_sel[3] = pick;
    }
    __syncthreads();
    if (tid == 0) {
        int pick = s_sel[3];
        if (pick < 0) {                 // rounding left the target at / beyond the total: the last kept token
            for (int i = V - 1; i >= 0; --i)
                if ((int)bf16_key(lr[i]) >= p_key) { pick = i; break; }
        }
        ids_out[row] = (int64_t)pick;
        counters[row] = (int32_t)(ctr + 1u);
        if (LOG && last_cta_out((unsigned*)lg.col + 1)) {
            lg.col[0] += 1;
            __threadfence();
        }
    }
}

// ================================================================================================ speculative sampling
// Leviathan et al., Algorithm 1 (HF ``_speculative_sampling``) after a verify pass: the target's K+1 rows p_0..p_K and the
// assistant's K rows q_0..q_{K-1}, each warped by the rules above (tl_sample's kept set and weights), drafts d_i =
// in_ids[i+1] drawn from q_i.  Two launches:
//   * spec_rows_kernel  one CTA per row (2K+1, in parallel): row_analysis -> SpecRow in the workspace
//   * spec_draw_kernel  one CTA: draft i < n_cand is kept while u_i * q_i(d_i) < p_i(d_i) (u_i = Philox row i); at the
//                       first rejection n the token is drawn from (p_n - q_n)+ without d_n, else from p_n (Philox row
//                       SPEC_DRAW_ROW), by the inverse CDF in index order with fixed-order sums
// Every probability is weight / Z_kept of its row, in double.  An id >= V_q has q = 0; a draft >= V_p has p = 0 and is
// always rejected; ids >= V_p carry no residual mass, so the draw runs over 0..V_p-1.
struct SpecRow {
    float x_max;
    int p_key;
    double Z;
};
constexpr int SPEC_DRAW_ROW = 16;       // Philox row of the final draw; the acceptance uniforms take rows 0..K-1 (K <= 15)

__device__ __forceinline__ double kept_weight(const uint16_t* lr, int t, const SpecRow& s, float inv_temp) {
    const uint32_t key = bf16_key(lr[t]);
    return (int)key >= s.p_key ? (double)__expf(key_value(key) * inv_temp - s.x_max) : 0.0;
}

__global__ void __launch_bounds__(SM_THREADS) spec_rows_kernel(const bf16* __restrict__ p_logits, int V_p,
                                                               const bf16* __restrict__ q_logits, int V_q, int K, float inv_temp,
                                                               int top_k, float top_p, SpecRow* __restrict__ rows,
                                                               uint32_t* __restrict__ hist_all) {
    const int r = blockIdx.x;                        // 0..K: p rows, K+1..2K: q rows
    const bool is_p = r <= K;
    const int V = is_p ? V_p : V_q;
    const uint16_t* lr = reinterpret_cast<const uint16_t*>(is_p ? p_logits : q_logits) + (size_t)(is_p ? r : r - K - 1) * V;
    __shared__ double s_warp[32];
    __shared__ int s_sel[4];
    __shared__ double s_val[2];
    const RowStats rs = row_analysis(lr, V, inv_temp, top_k, top_p, hist_all + (size_t)r * SM_BINS, s_warp, s_sel, s_val);
    if (threadIdx.x == 0) rows[r] = SpecRow{rs.x_max, rs.p_key, rs.Z_kept};
}

__global__ void __launch_bounds__(SM_THREADS) spec_draw_kernel(const bf16* __restrict__ p_logits, int V_p,
                                                               const bf16* __restrict__ q_logits, int V_q, int K,
                                                               const int64_t* __restrict__ in_ids, const int32_t* __restrict__ n_cand,
                                                               float inv_temp, unsigned long long seed, int32_t* __restrict__ counter,
                                                               const SpecRow* __restrict__ rows, int64_t* __restrict__ ids_out) {
    const int tid = threadIdx.x;
    const uint16_t* P = reinterpret_cast<const uint16_t*>(p_logits);
    const uint16_t* Q = reinterpret_cast<const uint16_t*>(q_logits);
    __shared__ double s_warp[32];
    __shared__ int s_n, s_pick;
    const uint32_t ctr = (uint32_t)*counter;
    const int nc = max(0, min(*n_cand, K));
    if (tid == 0) {
        int n = 0;
        for (; n < nc; ++n) {
            const int64_t d = in_ids[n + 1];
            const SpecRow &sp = rows[n], &sq = rows[K + 1 + n];
            const double p = d >= 0 && d < V_p ? kept_weight(P + (size_t)n * V_p, (int)d, sp, inv_temp) / sp.Z : 0.0;
            const double q = d >= 0 && d < V_q ? kept_weight(Q + (size_t)n * V_q, (int)d, sq, inv_temp) / sq.Z : 0.0;
            // strict: u can be 0, and a token the target's warpers removed (p = 0) must never be kept
            if (!((double)philox_uniform(seed, (uint32_t)n, ctr) * q < p)) break;
        }
        s_n = n;
        s_pick = -1;
    }
    __syncthreads();
    const int n = s_n;
    const bool resid = n < nc;
    const int64_t d = resid ? in_ids[n + 1] : -1;    // the rejected draft: never drawn, whatever the rounding
    const uint16_t* pr = P + (size_t)n * V_p;
    const uint16_t* qr = Q + (size_t)(resid ? n : 0) * V_q;
    const SpecRow sp = rows[n], sq = rows[K + 1 + (resid ? n : 0)];
    // resid: (p_n - q_n)+ in probabilities; otherwise p_n's kept weights (also the fallback when the residual mass is 0)
    auto weight = [&](int t, bool res) -> double {
        if (t == d) return 0.0;
        const double wp = kept_weight(pr, t, sp, inv_temp);
        if (!res) return wp;
        const double wq = t < V_q ? kept_weight(qr, t, sq, inv_temp) / sq.Z : 0.0;
        return fmax(0.0, wp / sp.Z - wq);
    };
    const double u = (double)philox_uniform(seed, (uint32_t)SPEC_DRAW_ROW, ctr);
    const int per = (V_p + SM_THREADS - 1) / SM_THREADS;
    const int i0 = tid * per, i1 = min(V_p, i0 + per);
    bool res = resid;
    double local_w, W, w_before;
    for (;;) {
        local_w = 0.0;
        for (int i = i0; i < i1; ++i) local_w += weight(i, res);
        w_before = block_excl_scan(local_w, s_warp, &W);
        if (W > 0.0 || !res) break;
        res = false;                                 // the residual rounded to 0 (p_n == q_n): draw from p_n
    }
    const double target = u * W;
    if (local_w > 0.0 && w_before <= target && target < w_before + local_w) {
        double c = w_before;
        int pick = -1;
        for (int i = i0; i < i1; ++i) {
            const double w = weight(i, res);
            if (w <= 0.0) continue;
            pick = i;
            c += w;
            if (target < c) break;
        }
        s_pick = pick;
    }
    __syncthreads();
    if (tid == 0) {
        int pick = s_pick;
        if (pick < 0) {                 // rounding left the target at / beyond the total: the last token of positive weight
            for (int i = V_p - 1; i >= 0; --i)
                if (weight(i, res) > 0.0) { pick = i; break; }
        }
        for (int i = 0; i < n; ++i) ids_out[i] = in_ids[i + 1];
        ids_out[n] = (int64_t)pick;
        *counter = (int32_t)(ctr + 1u);
    }
}

// ================================================================================================ processed sampling
// After the logits processors (logits_process.cu) a value is an arbitrary fp32, no longer one of 65536 bf16 patterns, so
// the rules above run on 32-bit monotone keys: a histogram of the high 16 key bits finds the boundary bin, and a second
// pass over the elements of that bin finds the boundary key.  Probability mass is summed as 64-bit fixed-point integers
// (2^40 = the row's maximum), so every sum is exact and independent of the order the atomics land in.
typedef unsigned long long u64;
constexpr double SP_ONE = 1099511627776.0;       // 2^40

__device__ __forceinline__ uint32_t f32_key(float v) {     // monotone; -0 and +0 share the key of +0
    const uint32_t b = __float_as_uint(v == 0.f ? 0.f : v);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_f32(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
__device__ __forceinline__ u64 key_weight(uint32_t key, float inv_temp, float x_max) {
    return (u64)((double)expf(key_f32(key) * inv_temp - x_max) * SP_ONE);
}

__device__ u64 block_excl_scan_u64(u64 v, u64* s_warp, u64* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    u64 x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const u64 y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
        u64 w = s_warp[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const u64 y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        s_warp[lane] = w;
    }
    __syncthreads();
    const u64 before = (warp ? s_warp[warp - 1] : 0ull) + (x - v);
    *total = s_warp[31];
    __syncthreads();
    return before;
}

struct Crossing { int bin; u64 above, T; };

// Walking the 65536 bins of h downwards: the bin b with above(b) < T <= above(b) + h[b], where above(b) is the sum of the
// bins over b and T = T_abs, or ceil(frac * total) when frac >= 0.  All comparisons are integer: exactly one bin.
__device__ Crossing find_crossing(const u64* h, u64 T_abs, float frac, u64* s_warp, Crossing* s_out) {
    const int hi = SM_BINS - 1 - (int)threadIdx.x * SM_PER;
    u64 local = 0;
    for (int j = 0; j < SM_PER; ++j) local += h[hi - j];
    u64 total;
    const u64 before = block_excl_scan_u64(local, s_warp, &total);
    const u64 T = frac < 0.f ? T_abs : (u64)ceil((double)frac * (double)total);
    if (before < T && T <= before + local) {
        u64 c = before;
        for (int j = 0; j < SM_PER; ++j) {
            const u64 x = h[hi - j];
            if (c + x >= T) { *s_out = Crossing{hi - j, c, T}; break; }
            c += x;
        }
    }
    __syncthreads();
    const Crossing r = *s_out;
    __syncthreads();
    return r;
}

__device__ __forceinline__ void clear_bins(u64* h) {
    for (int i = threadIdx.x; i < SM_BINS; i += SM_THREADS) h[i] = 0ull;
    __syncthreads();
}

// LOG: as sample_kernel's, over the processed values (-inf for a banned id stays -inf)
template <bool LOG = false>
__global__ void __launch_bounds__(SM_THREADS) sample_proc_kernel(const bf16* __restrict__ logits, int64_t* __restrict__ ids_out,
                                                                 int V, LpRows h, float inv_temp, int top_k, float top_p,
                                                                 unsigned long long seed, int32_t* __restrict__ counters,
                                                                 u64* __restrict__ hist_all, LogDesc lg) {
    const int row = blockIdx.x, tid = threadIdx.x;
    const bf16* lr = logits + (size_t)row * V;
    const uint32_t* bits = h.bits + (size_t)row * h.W;
    const uint32_t* ban = h.ban ? h.ban + (size_t)row * h.W : nullptr;
    const float penalty = __int_as_float(h.params[TL_LP_PENALTY]);
    u64* hist = hist_all + (size_t)row * SM_BINS;
    __shared__ u64 s_warp[32];
    __shared__ float s_max[32];
    __shared__ Crossing s_cross;
    __shared__ int s_pick;
    auto key_at = [&](int i) { return f32_key(lp_value(bf2f(lr[i]), i, bits, ban, penalty)); };
    const bool use_k = top_k > 0 && top_k < V;
    // ---- max (and the top-k count histogram of the high key bits)
    if (use_k) clear_bins(hist);
    float vmax = -INFINITY;
    for (int i = tid; i < V; i += SM_THREADS) {
        const uint32_t key = key_at(i);
        vmax = fmaxf(vmax, key_f32(key));
        if (use_k) atomicAdd(&hist[key >> 16], 1ull);
    }
    vmax = warp_max(vmax);
    if ((tid & 31) == 0) s_max[tid >> 5] = vmax;
    __syncthreads();
    vmax = warp_max(s_max[tid & 31]);
    const uint32_t ctr = (uint32_t)counters[row];
    float *raw = nullptr, *proc = nullptr;
    const bool log = LOG && log_rows(lg, *lg.col, row, V, &raw, &proc);
    if (vmax == -INFINITY) {                  // every token banned: token 0, as the argmax returns
        if (LOG && log) {
            for (int i = tid; i < V; i += SM_THREADS) {
                if (raw) raw[i] = bf2f(lr[i]);
                if (proc) proc[i] = -INFINITY;
            }
        }
        if (LOG) __syncthreads();
        if (tid == 0) {
            ids_out[row] = 0;
            counters[row] = (int32_t)(ctr + 1u);
            lp_append(h, row, 0);
            if (LOG && last_cta_out((unsigned*)lg.col + 1)) {
                lg.col[0] += 1;
                __threadfence();
            }
        }
        return;
    }
    const float x_max = vmax * inv_temp;
    // ---- top-k: the key of the k-th largest value; every value >= it is kept
    uint32_t k_key = 0;
    if (use_k) {
        const Crossing c = find_crossing(hist, (u64)top_k, -1.f, s_warp, &s_cross);
        clear_bins(hist);
        for (int i = tid; i < V; i += SM_THREADS) {
            const uint32_t key = key_at(i);
            if ((int)(key >> 16) == c.bin) atomicAdd(&hist[key & 0xffffu], 1ull);
        }
        __syncthreads();
        const Crossing lo = find_crossing(hist, c.T - c.above, -1.f, s_warp, &s_cross);
        k_key = ((uint32_t)c.bin << 16) | (uint32_t)lo.bin;
    }
    // ---- top-p: the lowest key whose mass above is < top_p * Z (its whole tie group is kept)
    uint32_t p_key = k_key;
    if (top_p < 1.0f) {
        clear_bins(hist);
        for (int i = tid; i < V; i += SM_THREADS) {
            const uint32_t key = key_at(i);
            if (key >= k_key) atomicAdd(&hist[key >> 16], key_weight(key, inv_temp, x_max));
        }
        __syncthreads();
        const Crossing c = find_crossing(hist, 0ull, top_p, s_warp, &s_cross);
        clear_bins(hist);
        for (int i = tid; i < V; i += SM_THREADS) {
            const uint32_t key = key_at(i);
            if (key >= k_key && (int)(key >> 16) == c.bin) atomicAdd(&hist[key & 0xffffu], key_weight(key, inv_temp, x_max));
        }
        __syncthreads();
        const Crossing lo = find_crossing(hist, c.T - c.above, -1.f, s_warp, &s_cross);
        p_key = ((uint32_t)c.bin << 16) | (uint32_t)lo.bin;
    }
    // ---- draw and invert the CDF over the kept tokens in index order (integer prefix sums: exact)
    const int per = (V + SM_THREADS - 1) / SM_THREADS;
    const int i0 = tid * per, i1 = min(V, i0 + per);
    if (LOG && log) {
        for (int i = tid; i < V; i += SM_THREADS) {          // interleaved, not the draw's per-thread ranges: coalesced stores
            const float x = bf2f(lr[i]), v = lp_value(x, i, bits, ban, penalty);
            if (raw) raw[i] = x;
            if (proc) proc[i] = f32_key(v) >= p_key ? __fdiv_rn(v, lg.temperature) : -INFINITY;
        }
    }
    u64 local_w = 0;
    for (int i = i0; i < i1; ++i) {
        const uint32_t key = key_at(i);
        if (key >= p_key) local_w += key_weight(key, inv_temp, x_max);
    }
    if (tid == 0) s_pick = -1;
    u64 W;
    const u64 w_before = block_excl_scan_u64(local_w, s_warp, &W);
    const u64 target = min(W - 1, (u64)((double)philox_uniform(seed, (uint32_t)row, ctr) * (double)W));
    if (local_w > 0 && w_before <= target && target < w_before + local_w) {
        u64 c = w_before;
        for (int i = i0; i < i1; ++i) {
            const uint32_t key = key_at(i);
            if (key < p_key) continue;
            c += key_weight(key, inv_temp, x_max);
            if (target < c) { s_pick = i; break; }
        }
    }
    __syncthreads();
    if (tid == 0) {
        const int pick = s_pick < 0 ? 0 : s_pick;
        ids_out[row] = (int64_t)pick;
        counters[row] = (int32_t)(ctr + 1u);
        lp_append(h, row, pick);
        if (LOG && last_cta_out((unsigned*)lg.col + 1)) {
            lg.col[0] += 1;
            __threadfence();
        }
    }
}

}  // namespace tl

extern "C" {

static int sample_proc_launch(const void* logits, int64_t* ids_out, int32_t* log, int32_t* len, uint32_t* bits,
                              const int32_t* params_dev, int flags, int M, int V, int L, float temperature, int top_k, float top_p,
                              unsigned long long seed, int32_t* counters_dev, void* workspace, size_t ws_bytes,
                              const tl::LogDesc* lg, void* stream) {
    using namespace tl;
    TL_REQUIRE(logits && ids_out && log && len && bits && params_dev && counters_dev && workspace, TL_ERR_INVALID,
               "tl_sample_proc: null argument");
    TL_REQUIRE(M >= 1 && V >= 1 && L >= 1, TL_ERR_INVALID, "tl_sample_proc: bad shape M=%d V=%d L=%d", M, V, L);
    TL_REQUIRE(temperature > 0.f && top_p > 0.f && top_p <= 1.f && top_k >= 0, TL_ERR_INVALID,
               "tl_sample_proc: temperature must be > 0, 0 < top_p <= 1, top_k >= 0 (got %g, %g, %d)", temperature, top_p, top_k);
    TL_REQUIRE(ws_bytes >= tl_logits_proc_ws(M, V), TL_ERR_WORKSPACE, "tl_sample_proc: workspace %zu < %zu", ws_bytes,
               tl_logits_proc_ws(M, V));
    cudaStream_t st = (cudaStream_t)stream;
    uint32_t* ban = (uint32_t*)workspace;
    const LpRows h{log, len, bits, (flags & TL_LP_BAN) ? ban : nullptr, params_dev, L, lp_words(V)};
    if (flags & TL_LP_BAN) {
        const int rc = lp_ban_launch(h, ban, M, V, st);
        if (rc != TL_OK) return rc;
    }
    u64* hist = (u64*)((unsigned char*)workspace + lp_ban_bytes(M, V));
    if (lg)
        sample_proc_kernel<true><<<M, SM_THREADS, 0, st>>>((const bf16*)logits, ids_out, V, h, 1.0f / temperature, top_k, top_p, seed,
                                                           counters_dev, hist, *lg);
    else
        sample_proc_kernel<<<M, SM_THREADS, 0, st>>>((const bf16*)logits, ids_out, V, h, 1.0f / temperature, top_k, top_p, seed,
                                                     counters_dev, hist, LogDesc{});
    return check_launch("tl_sample_proc");
}

int tl_sample_proc(const void* logits, int64_t* ids_out, int32_t* log, int32_t* len, uint32_t* bits,
                   const int32_t* params_dev, int flags, int M, int V, int L, float temperature, int top_k, float top_p,
                   unsigned long long seed, int32_t* counters_dev, void* workspace, size_t ws_bytes, void* stream) {
    return sample_proc_launch(logits, ids_out, log, len, bits, params_dev, flags, M, V, L, temperature, top_k, top_p, seed,
                              counters_dev, workspace, ws_bytes, nullptr, stream);
}

int tl_sample_proc_log(const void* logits, int64_t* ids_out, int32_t* log, int32_t* len, uint32_t* bits,
                       const int32_t* params_dev, int flags, int M, int V, int L, float temperature, int top_k, float top_p,
                       unsigned long long seed, int32_t* counters_dev, void* workspace, size_t ws_bytes, float* raw_log,
                       float* score_log, int32_t* log_col, int n_cols, int B_total, int row0, void* stream) {
    using namespace tl;
    LogDesc lg;
    const int rc = make_log("tl_sample_proc_log", raw_log, score_log, log_col, n_cols, B_total, row0, M, V, temperature, &lg);
    if (rc != TL_OK) return rc;
    return sample_proc_launch(logits, ids_out, log, len, bits, params_dev, flags, M, V, L, temperature, top_k, top_p, seed,
                              counters_dev, workspace, ws_bytes, &lg, stream);
}

size_t tl_sample_ws(int M) { return (size_t)(M > 0 ? M : 0) * tl::SM_BINS * sizeof(uint32_t); }

static int sample_launch(const void* logits, int64_t* ids_out, int M, int V, float temperature, int top_k, float top_p,
                         unsigned long long seed, int32_t* counters_dev, void* workspace, size_t ws_bytes, const tl::LogDesc* lg,
                         void* stream) {
    using namespace tl;
    TL_REQUIRE(logits && ids_out && counters_dev && workspace, TL_ERR_INVALID, "tl_sample: null argument");
    TL_REQUIRE(M >= 1 && V >= 1, TL_ERR_INVALID, "tl_sample: bad shape M=%d V=%d", M, V);
    TL_REQUIRE(temperature > 0.f && top_p > 0.f && top_p <= 1.f && top_k >= 0, TL_ERR_INVALID,
               "tl_sample: temperature must be > 0, 0 < top_p <= 1, top_k >= 0 (got %g, %g, %d)", temperature, top_p, top_k);
    TL_REQUIRE(ws_bytes >= tl_sample_ws(M), TL_ERR_INVALID, "tl_sample: workspace too small");
    if (lg)
        sample_kernel<true><<<M, SM_THREADS, 0, (cudaStream_t)stream>>>((const bf16*)logits, ids_out, V, 1.0f / temperature, top_k,
                                                                        top_p, seed, counters_dev, (uint32_t*)workspace, *lg);
    else
        sample_kernel<<<M, SM_THREADS, 0, (cudaStream_t)stream>>>((const bf16*)logits, ids_out, V, 1.0f / temperature, top_k, top_p,
                                                                  seed, counters_dev, (uint32_t*)workspace, LogDesc{});
    return check_launch("tl_sample");
}

int tl_sample(const void* logits, int64_t* ids_out, int M, int V, float temperature, int top_k, float top_p,
              unsigned long long seed, int32_t* counters_dev, void* workspace, size_t ws_bytes, void* stream) {
    return sample_launch(logits, ids_out, M, V, temperature, top_k, top_p, seed, counters_dev, workspace, ws_bytes, nullptr, stream);
}

int tl_sample_log(const void* logits, int64_t* ids_out, int M, int V, float temperature, int top_k, float top_p,
                  unsigned long long seed, int32_t* counters_dev, void* workspace, size_t ws_bytes, float* raw_log,
                  float* score_log, int32_t* log_col, int n_cols, int B_total, int row0, void* stream) {
    using namespace tl;
    LogDesc lg;
    const int rc = make_log("tl_sample_log", raw_log, score_log, log_col, n_cols, B_total, row0, M, V, temperature, &lg);
    if (rc != TL_OK) return rc;
    return sample_launch(logits, ids_out, M, V, temperature, top_k, top_p, seed, counters_dev, workspace, ws_bytes, &lg, stream);
}

size_t tl_spec_accept_ws(int K) {
    const size_t rows = (size_t)(K > 0 ? 2 * K + 1 : 0);
    return rows * tl::SM_BINS * sizeof(uint32_t) + rows * sizeof(tl::SpecRow);
}

int tl_spec_accept(const void* p_logits, int V_p, const void* q_logits, int V_q, int K, const int64_t* in_ids,
                   const int32_t* n_cand, float temperature, int top_k, float top_p, unsigned long long seed,
                   int32_t* counter_dev, int64_t* ids_out, void* workspace, size_t ws_bytes, void* stream) {
    using namespace tl;
    TL_REQUIRE(p_logits && q_logits && in_ids && n_cand && counter_dev && ids_out && workspace, TL_ERR_INVALID,
               "tl_spec_accept: null argument");
    TL_REQUIRE(K >= 1 && K <= TL_PL_MAX_DRAFT && V_p >= 1 && V_q >= 1, TL_ERR_INVALID,
               "tl_spec_accept: bad shape K=%d V_p=%d V_q=%d", K, V_p, V_q);
    TL_REQUIRE(temperature > 0.f && top_p > 0.f && top_p <= 1.f && top_k >= 0, TL_ERR_INVALID,
               "tl_spec_accept: temperature must be > 0, 0 < top_p <= 1, top_k >= 0 (got %g, %g, %d)", temperature, top_p, top_k);
    TL_REQUIRE(ws_bytes >= tl_spec_accept_ws(K), TL_ERR_INVALID, "tl_spec_accept: workspace %zu < %zu", ws_bytes,
               tl_spec_accept_ws(K));
    cudaStream_t st = (cudaStream_t)stream;
    uint32_t* hist = (uint32_t*)workspace;
    SpecRow* rows = (SpecRow*)(hist + (size_t)(2 * K + 1) * SM_BINS);
    const float inv_temp = 1.0f / temperature;
    spec_rows_kernel<<<2 * K + 1, SM_THREADS, 0, st>>>((const bf16*)p_logits, V_p, (const bf16*)q_logits, V_q, K, inv_temp, top_k,
                                                       top_p, rows, hist);
    const int rc = check_launch("tl_spec_accept");
    if (rc != TL_OK) return rc;
    spec_draw_kernel<<<1, SM_THREADS, 0, st>>>((const bf16*)p_logits, V_p, (const bf16*)q_logits, V_q, K, in_ids, n_cand, inv_temp,
                                               seed, counter_dev, rows, ids_out);
    return check_launch("tl_spec_accept");
}

}  // extern "C"
