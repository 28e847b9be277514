// Token sampling on the device: temperature -> top-k -> top-p -> min-p -> typical -> epsilon -> eta -> multinomial draw,
// one CTA per row.
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
//
// HF's remaining warpers (MinP, Typical, Epsilon, Eta; min_tokens_to_keep = 1) each act on the set the stages before them
// kept, with p = softmax(x / T) over that set:
//   * min_p              keep p >= min_p * p_max (the set's top tie group always stays; min_p = 1 keeps only it)
//   * typical_p = m      c = lse - H (H: the set's entropy) = E[x/T]; rank by the distance |c - x/T| and keep a distance
//                        group while the mass of the strictly closer tokens is < m: top-p on the key -distance
//   * epsilon_cutoff     keep p >= eps, and every token >= the set's top value
//   * eta_cutoff         the same with eps = min(eta, sqrt(eta) * exp(-H))
// Every one of them keeps ONE interval of keys, so the kept set is always [lo_key, hi_key]; typical may drop the top
// tokens, which is why hi_key exists.  After typical the weights are rebased on the new top (x_ref = value(hi_key) / T),
// so the kept mass never rounds to zero however far below the row's max the band lies: the top kept token weighs ~1.
// The distance is ranked as the fp32 value |E[a] - a| (a = x/T - x_ref), so equal fp32 distances form one group.
// These stages run only in the WARP instantiations, which the host selects when one of them is on; the others are the
// kernels as they were.
#include "common.cuh"

namespace tl {

constexpr int SM_THREADS = 1024;
constexpr int SM_BINS = 65536;
constexpr int SM_PER = SM_BINS / SM_THREADS;      // bins per thread in the scans
static_assert(SM_PER == 64, "the warpers' occupancy mask holds one thread's bins in 64 bits");

__device__ __forceinline__ uint32_t bf16_key(uint16_t bits) {       // monotone: larger value -> larger key
    return (bits & 0x8000u) ? (uint32_t)(uint16_t)~bits : (uint32_t)(bits | 0x8000u);
}
__device__ __forceinline__ float key_value(uint32_t key) {
    const uint16_t bits = (key & 0x8000u) ? (uint16_t)(key & 0x7fffu) : (uint16_t)~key;
    return __uint_as_float(((uint32_t)bits) << 16);
}

// min_p, typical_p, epsilon_cutoff, eta_cutoff; off at (0, 1, 0, 0)
struct Warpers {
    float min_p, typical_p, epsilon, eta;
};
inline bool warpers_on(const Warpers& w) { return w.min_p > 0.f || w.typical_p < 1.f || w.epsilon > 0.f || w.eta > 0.f; }

// key in the kept set [lo, hi]; without the warpers the set is key >= lo
template <bool WARP, typename K>
__device__ __forceinline__ bool in_set(K key, K lo, K hi) {
    if constexpr (WARP) return key >= lo && key <= hi;
    else return key >= lo;
}

// the occupied bins of a thread's range [hk - SM_PER + 1, hk] that lie in [lo, hi], as a mask (bit j: key hk - j)
__device__ __forceinline__ unsigned long long bins_in(unsigned long long occ, int hk, int lo, int hi) {
    const int j0 = max(0, hk - hi), j1 = min(SM_PER - 1, hk - lo);
    if (j0 > j1) return 0ull;
    const int n = j1 - j0 + 1;
    return occ & ((n == 64 ? ~0ull : (1ull << n) - 1ull) << j0);
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
// WARP: then min_p, typical, epsilon and eta on the bins, every sum in double in a fixed order (each thread's occupied
// bins downwards, then the block scan in thread order).  Typical finds its radius by bisection on the fp32 bit pattern
// of the distance (monotone for distances >= 0): the smallest radius r whose mass within(r) = sum of the bins at
// distance <= r reaches typical_p * Z.  within() only grows with r (sums of non-negative terms in a fixed order), so the
// 31 steps find the crossing group's distance exactly; if rounding leaves within(inf) below the limit, the set stays.
struct RowStats {
    float x_max;        // the weights' reference: weight(key) = __expf(key_value(key) * inv_temp - x_max); the row's max
                        // logit / temperature, or with the warpers the top kept value / temperature
    int p_key;          // kept: key >= p_key (lo_key)
    double Z_kept;      // the kept mass, summed over the bins
    int hi_key;         // and key <= hi_key (WARP only; SM_BINS - 1 otherwise)
};

template <bool WARP = false>
__device__ __forceinline__ RowStats row_analysis(const uint16_t* __restrict__ lr, int V, float inv_temp, int top_k, float top_p,
                                                 uint32_t* __restrict__ hist, double* s_warp, int* s_sel, double* s_val,
                                                 Warpers wp = Warpers{0.f, 1.f, 0.f, 0.f}) {
    const int tid = threadIdx.x;
    for (int i = tid; i < SM_BINS; i += SM_THREADS) hist[i] = 0u;
    __syncthreads();
    for (int i = tid; i < V; i += SM_THREADS) atomicAdd(&hist[bf16_key(lr[i])], 1u);
    __syncthreads();
    // this thread owns bins [hi_key - SM_PER + 1, hi_key], walked downwards: thread 0 holds the largest values
    const int hi_key = SM_BINS - 1 - tid * SM_PER;
    // the bins' counts: a per-thread array, or with WARP read from hist again (the array would sit in local memory
    // beside the warpers' state)
    uint32_t cnt[SM_PER];
    auto count = [&](int j) -> uint32_t {
        if constexpr (WARP) return hist[hi_key - j];
        else return cnt[j];
    };
    uint32_t local_n = 0;
    unsigned long long occ = 0ull;                   // WARP: the occupied bins (bit j: key hi_key - j)
#pragma unroll 8
    for (int j = 0; j < SM_PER; ++j) {
        const uint32_t c = hist[hi_key - j];
        if constexpr (!WARP) cnt[j] = c;
        local_n += c;
        if constexpr (WARP) occ |= (unsigned long long)(c != 0u) << j;
    }
    // ---- max: the first occupied bin from the top
    double tot;
    const double n_before = block_excl_scan((double)local_n, s_warp, &tot);
    if (n_before == 0.0 && local_n > 0) {
        for (int j = 0; j < SM_PER; ++j)
            if (count(j)) { s_sel[0] = hi_key - j; break; }
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
                c += (double)count(j);
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
        if (count(j) && key >= k_key) local_m += (double)count(j) * (double)__expf(key_value((uint32_t)key) * inv_temp - x_max);
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
                if (!(count(j) && key >= k_key)) continue;
                const double w = (double)count(j) * (double)__expf(key_value((uint32_t)key) * inv_temp - x_max);
                if (c < lim) { s_sel[2] = key; s_val[0] = c + w; }     // kept: mass above it is still below the limit
                c += w;
            }
        }
        __syncthreads();
        p_key = s_sel[2];
        Z_kept = s_val[0];
    }
    if constexpr (!WARP) {
        return RowStats{x_max, p_key, Z_kept, SM_BINS - 1};
    } else {
        __shared__ int s_key[2];
        int lo = p_key, hi = max_key;
        float x_ref = x_max;
        auto wgt = [&](int key) { return key_value((uint32_t)key) * inv_temp - x_ref; };    // a = x/T - x_ref
        // the mass of [lo, hi] and, with wa, the sum of weight * a over the tokens of positive weight (a -inf logit
        // weighs 0 and its a is -inf: 0 * -inf would be NaN; HF's entropies leave such tokens out too)
        auto mass = [&](double* wa) -> double {
            double m = 0.0, ma = 0.0;
            for (unsigned long long b = bins_in(occ, hi_key, lo, hi); b; b &= b - 1ull) {
                const int key = hi_key - (__ffsll((long long)b) - 1);
                const float a = wgt(key);
                const double w = (double)hist[key] * (double)__expf(a);
                m += w;
                if (w > 0.0) ma += w * (double)a;
            }
            double Z, WA;
            block_excl_scan(m, s_warp, &Z);
            if (wa) {
                block_excl_scan(ma, s_warp, &WA);
                *wa = WA;
            }
            return Z;
        };
        // the lowest key of [lo, hi] whose per-token weight is >= t (weights grow with the key), else hi
        auto lowest = [&](double t) -> int {
            __syncthreads();
            if (tid == 0) s_key[0] = hi;
            __syncthreads();
            int best = hi;
            for (unsigned long long b = bins_in(occ, hi_key, lo, hi); b; b &= b - 1ull) {
                const int key = hi_key - (__ffsll((long long)b) - 1);
                if (!((double)__expf(wgt(key)) >= t)) break;
                best = key;
            }
            atomicMin(&s_key[0], best);
            __syncthreads();
            return s_key[0];
        };
        double Z = Z_kept;
        if (wp.min_p > 0.f) {
            lo = lowest((double)wp.min_p * (double)__expf(wgt(hi)));
            Z = mass(nullptr);
        }
        if (wp.typical_p < 1.f) {
            double WA;
            Z = mass(&WA);
            const double mean = WA / Z, lim = (double)wp.typical_p * Z;
            auto dist = [&](int key) { return __float_as_uint((float)fabs(mean - (double)wgt(key))); };
            auto within = [&](uint32_t r) -> double {
                double m = 0.0, tot;
                for (unsigned long long b = bins_in(occ, hi_key, lo, hi); b; b &= b - 1ull) {
                    const int key = hi_key - (__ffsll((long long)b) - 1);
                    if (dist(key) <= r) m += (double)hist[key] * (double)__expf(wgt(key));
                }
                block_excl_scan(m, s_warp, &tot);
                return tot;
            };
            uint32_t r_lo = 0u, r_hi = 0x7f800000u;      // +inf: everything
            if (within(r_hi) >= lim) {
                while (r_lo < r_hi) {
                    const uint32_t mid = r_lo + (r_hi - r_lo) / 2u;
                    if (within(mid) >= lim) r_hi = mid;
                    else r_lo = mid + 1u;
                }
            }
            if (tid == 0) { s_key[0] = hi; s_key[1] = lo; }
            __syncthreads();
            int kmin = hi, kmax = lo;
            for (unsigned long long b = bins_in(occ, hi_key, lo, hi); b; b &= b - 1ull) {
                const int key = hi_key - (__ffsll((long long)b) - 1);
                if (dist(key) <= r_hi) { kmin = min(kmin, key); kmax = max(kmax, key); }
            }
            atomicMin(&s_key[0], kmin);
            atomicMax(&s_key[1], kmax);
            __syncthreads();
            lo = s_key[0];
            hi = s_key[1];
            x_ref = key_value((uint32_t)hi) * inv_temp;
            Z = mass(nullptr);
        }
        if (wp.epsilon > 0.f) {
            lo = lowest((double)wp.epsilon * Z);
            Z = mass(nullptr);
        }
        if (wp.eta > 0.f) {
            double WA;
            Z = mass(&WA);
            const double H = log(Z) - WA / Z;
            lo = lowest(fmin((double)wp.eta, sqrt((double)wp.eta) * exp(-H)) * Z);
            Z = mass(nullptr);
        }
        return RowStats{x_ref, lo, Z, hi};
    }
}

// LOG: once p_key is known, a pass over the row stores it into the score log (common.cuh LogDesc): the raw logit, and
// x / temperature on the kept set, -inf elsewhere.  The pass strides by the CTA's width, so its stores coalesce (the
// draw's per-thread ranges would scatter them).  The CTAs (rows) share the log column, so the last CTA out advances it.
// The draw itself does not depend on LOG.  WARP: the warpers after top-p (Warpers); the kept set is [p_key, hi_key].
template <bool LOG = false, bool WARP = false>
__global__ void __launch_bounds__(SM_THREADS) sample_kernel(const bf16* __restrict__ logits, int64_t* __restrict__ ids_out, int V,
                                                            float inv_temp, int top_k, float top_p, unsigned long long seed,
                                                            int32_t* __restrict__ counters, uint32_t* __restrict__ hist_all,
                                                            LogDesc lg, Warpers wp) {
    const int row = blockIdx.x, tid = threadIdx.x;
    const uint16_t* lr = reinterpret_cast<const uint16_t*>(logits) + (size_t)row * V;
    __shared__ double s_warp[32];
    __shared__ int s_sel[4];
    __shared__ double s_val[2];
    const auto [x_max, p_key, Z_kept, hi_key] = row_analysis<WARP>(lr, V, inv_temp, top_k, top_p, hist_all + (size_t)row * SM_BINS,
                                                                    s_warp, s_sel, s_val, wp);
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
            if (proc) proc[i] = in_set<WARP>((int)bf16_key(lr[i]), p_key, hi_key) ? __fdiv_rn(x, lg.temperature) : -INFINITY;
        }
    }
    double local_w = 0.0;
    for (int i = i0; i < i1; ++i) {
        const uint32_t key = bf16_key(lr[i]);
        if (in_set<WARP>((int)key, p_key, hi_key)) local_w += (double)__expf(key_value(key) * inv_temp - x_max);
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
            if (!in_set<WARP>((int)key, p_key, hi_key)) continue;
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
                if (in_set<WARP>((int)bf16_key(lr[i]), p_key, hi_key)) { pick = i; break; }
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
    int hi_key;
};
constexpr int SPEC_DRAW_ROW = 16;       // Philox row of the final draw; the acceptance uniforms take rows 0..K-1 (K <= 15)

template <bool WARP>
__device__ __forceinline__ double kept_weight(const uint16_t* lr, int t, const SpecRow& s, float inv_temp) {
    const uint32_t key = bf16_key(lr[t]);
    return in_set<WARP>((int)key, s.p_key, s.hi_key) ? (double)__expf(key_value(key) * inv_temp - s.x_max) : 0.0;
}

template <bool WARP = false>
__global__ void __launch_bounds__(SM_THREADS) spec_rows_kernel(const bf16* __restrict__ p_logits, int V_p,
                                                               const bf16* __restrict__ q_logits, int V_q, int K, float inv_temp,
                                                               int top_k, float top_p, SpecRow* __restrict__ rows,
                                                               uint32_t* __restrict__ hist_all, Warpers wp) {
    const int r = blockIdx.x;                        // 0..K: p rows, K+1..2K: q rows
    const bool is_p = r <= K;
    const int V = is_p ? V_p : V_q;
    const uint16_t* lr = reinterpret_cast<const uint16_t*>(is_p ? p_logits : q_logits) + (size_t)(is_p ? r : r - K - 1) * V;
    __shared__ double s_warp[32];
    __shared__ int s_sel[4];
    __shared__ double s_val[2];
    const RowStats rs = row_analysis<WARP>(lr, V, inv_temp, top_k, top_p, hist_all + (size_t)r * SM_BINS, s_warp, s_sel, s_val, wp);
    if (threadIdx.x == 0) rows[r] = SpecRow{rs.x_max, rs.p_key, rs.Z_kept, rs.hi_key};
}

template <bool WARP = false>
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
            const double p = d >= 0 && d < V_p ? kept_weight<WARP>(P + (size_t)n * V_p, (int)d, sp, inv_temp) / sp.Z : 0.0;
            const double q = d >= 0 && d < V_q ? kept_weight<WARP>(Q + (size_t)n * V_q, (int)d, sq, inv_temp) / sq.Z : 0.0;
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
        const double wp = kept_weight<WARP>(pr, t, sp, inv_temp);
        if (!res) return wp;
        const double wq = t < V_q ? kept_weight<WARP>(qr, t, sq, inv_temp) / sq.Z : 0.0;
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
// WARP: the warpers after top-p, each over the kept interval [lo, hi] by passes over the row: min_p, epsilon and eta
// compare each element's fixed-point weight with the threshold and take the block min of the keys that pass (the top
// key hi always stays); the entropy's sum of weight * a is a fixed-order double sum (each thread's elements in index
// order, then the block scan); typical is top-p over the distance key ~f32_key(|E[a] - a|) (closer: larger) through
// the same two-level find_crossing, and its new interval is the block min / max of the keys it keeps.  After typical
// the weights are rebased on the kept top (x_ref), which then weighs 2^40, so the kept mass is never 0.
template <bool LOG = false, bool WARP = false>
__global__ void __launch_bounds__(SM_THREADS) sample_proc_kernel(const bf16* __restrict__ logits, int64_t* __restrict__ ids_out,
                                                                 int V, LpRows h, float inv_temp, int top_k, float top_p,
                                                                 unsigned long long seed, int32_t* __restrict__ counters,
                                                                 u64* __restrict__ hist_all, LogDesc lg, Warpers wp) {
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
    uint32_t hi_key = 0xffffffffu;
    float x_ref = x_max;
    if constexpr (WARP) {
        __shared__ double s_wd[32];
        __shared__ uint32_t s_key[2];
        hi_key = f32_key(vmax);
        // the fixed-point mass of [p_key, hi_key] (exact) and, with wa, the fixed-order sum of weight * a
        auto mass = [&](double* wa) -> u64 {
            u64 m = 0;
            double ma = 0.0;
            for (int i = tid; i < V; i += SM_THREADS) {
                const uint32_t key = key_at(i);
                if (key < p_key || key > hi_key) continue;
                const u64 w = key_weight(key, inv_temp, x_ref);
                m += w;
                if (wa && w) ma += (double)w * (double)(key_f32(key) * inv_temp - x_ref);    // a banned id: w = 0, a = -inf
            }
            u64 Z;
            block_excl_scan_u64(m, s_warp, &Z);
            if (wa) {
                double WA;
                block_excl_scan(ma, s_wd, &WA);
                *wa = WA;
            }
            return Z;
        };
        // the lowest key of [p_key, hi_key] whose weight is >= t, else hi_key
        auto lowest = [&](double t) -> uint32_t {
            __syncthreads();
            if (tid == 0) s_key[0] = hi_key;
            __syncthreads();
            uint32_t best = hi_key;
            for (int i = tid; i < V; i += SM_THREADS) {
                const uint32_t key = key_at(i);
                if (key >= p_key && key < best && (double)key_weight(key, inv_temp, x_ref) >= t) best = key;
            }
            atomicMin(&s_key[0], best);
            __syncthreads();
            return s_key[0];
        };
        u64 Z = 0;
        if (wp.min_p > 0.f) p_key = lowest((double)wp.min_p * (double)key_weight(hi_key, inv_temp, x_ref));
        if (wp.typical_p < 1.f) {
            double WA;
            Z = mass(&WA);
            const double mean = WA / (double)Z;
            auto dkey = [&](uint32_t key) { return ~f32_key((float)fabs(mean - (double)(key_f32(key) * inv_temp - x_ref))); };
            clear_bins(hist);
            for (int i = tid; i < V; i += SM_THREADS) {
                const uint32_t key = key_at(i);
                if (key >= p_key && key <= hi_key) atomicAdd(&hist[dkey(key) >> 16], key_weight(key, inv_temp, x_ref));
            }
            __syncthreads();
            const Crossing c = find_crossing(hist, 0ull, wp.typical_p, s_warp, &s_cross);
            clear_bins(hist);
            for (int i = tid; i < V; i += SM_THREADS) {
                const uint32_t key = key_at(i);
                if (key >= p_key && key <= hi_key && (int)(dkey(key) >> 16) == c.bin)
                    atomicAdd(&hist[dkey(key) & 0xffffu], key_weight(key, inv_temp, x_ref));
            }
            __syncthreads();
            const Crossing l = find_crossing(hist, c.T - c.above, -1.f, s_warp, &s_cross);
            const uint32_t d_key = ((uint32_t)c.bin << 16) | (uint32_t)l.bin;
            if (tid == 0) { s_key[0] = hi_key; s_key[1] = p_key; }
            __syncthreads();
            uint32_t kmin = hi_key, kmax = p_key;
            for (int i = tid; i < V; i += SM_THREADS) {
                const uint32_t key = key_at(i);
                if (key >= p_key && key <= hi_key && dkey(key) >= d_key) { kmin = min(kmin, key); kmax = max(kmax, key); }
            }
            atomicMin(&s_key[0], kmin);
            atomicMax(&s_key[1], kmax);
            __syncthreads();
            p_key = s_key[0];
            hi_key = s_key[1];
            x_ref = key_f32(hi_key) * inv_temp;
        }
        if (wp.epsilon > 0.f) {
            Z = mass(nullptr);
            p_key = lowest((double)wp.epsilon * (double)Z);
        }
        if (wp.eta > 0.f) {
            double WA;
            Z = mass(&WA);
            const double H = ::log((double)Z / SP_ONE) - WA / (double)Z;
            p_key = lowest(fmin((double)wp.eta, sqrt((double)wp.eta) * exp(-H)) * (double)Z);
        }
    }
    // ---- draw and invert the CDF over the kept tokens in index order (integer prefix sums: exact)
    const int per = (V + SM_THREADS - 1) / SM_THREADS;
    const int i0 = tid * per, i1 = min(V, i0 + per);
    if (LOG && log) {
        for (int i = tid; i < V; i += SM_THREADS) {          // interleaved, not the draw's per-thread ranges: coalesced stores
            const float x = bf2f(lr[i]), v = lp_value(x, i, bits, ban, penalty);
            if (raw) raw[i] = x;
            if (proc) proc[i] = in_set<WARP>(f32_key(v), p_key, hi_key) ? __fdiv_rn(v, lg.temperature) : -INFINITY;
        }
    }
    u64 local_w = 0;
    for (int i = i0; i < i1; ++i) {
        const uint32_t key = key_at(i);
        if (in_set<WARP>(key, p_key, hi_key)) local_w += key_weight(key, inv_temp, x_ref);
    }
    if (tid == 0) s_pick = -1;
    u64 W;
    const u64 w_before = block_excl_scan_u64(local_w, s_warp, &W);
    const u64 target = min(W - 1, (u64)((double)philox_uniform(seed, (uint32_t)row, ctr) * (double)W));
    if (local_w > 0 && w_before <= target && target < w_before + local_w) {
        u64 c = w_before;
        for (int i = i0; i < i1; ++i) {
            const uint32_t key = key_at(i);
            if (!in_set<WARP>(key, p_key, hi_key)) continue;
            c += key_weight(key, inv_temp, x_ref);
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

// the warpers' ranges (0 / 1 = off): min_p in [0, 1], typical_p in (0, 1], epsilon and eta in [0, 1)
static int check_warpers(const char* what, float min_p, float typical_p, float epsilon, float eta, tl::Warpers* w) {
    TL_REQUIRE(min_p >= 0.f && min_p <= 1.f && typical_p > 0.f && typical_p <= 1.f && epsilon >= 0.f && epsilon < 1.f &&
                   eta >= 0.f && eta < 1.f, TL_ERR_INVALID,
               "%s: need 0 <= min_p <= 1, 0 < typical_p <= 1, 0 <= epsilon < 1, 0 <= eta < 1 (got %g, %g, %g, %g)", what, min_p,
               typical_p, epsilon, eta);
    *w = tl::Warpers{min_p, typical_p, epsilon, eta};
    return TL_OK;
}

static int sample_proc_launch(const void* logits, int64_t* ids_out, int32_t* log, int32_t* len, uint32_t* bits,
                              const int32_t* params_dev, int flags, int M, int V, int L, float temperature, int top_k, float top_p,
                              unsigned long long seed, int32_t* counters_dev, void* workspace, size_t ws_bytes,
                              const tl::LogDesc* lg, void* stream, float min_p, float typical_p, float epsilon, float eta) {
    using namespace tl;
    TL_REQUIRE(logits && ids_out && log && len && bits && params_dev && counters_dev && workspace, TL_ERR_INVALID,
               "tl_sample_proc: null argument");
    TL_REQUIRE(M >= 1 && V >= 1 && L >= 1, TL_ERR_INVALID, "tl_sample_proc: bad shape M=%d V=%d L=%d", M, V, L);
    TL_REQUIRE(temperature > 0.f && top_p > 0.f && top_p <= 1.f && top_k >= 0, TL_ERR_INVALID,
               "tl_sample_proc: temperature must be > 0, 0 < top_p <= 1, top_k >= 0 (got %g, %g, %d)", temperature, top_p, top_k);
    Warpers wp;
    int rc = check_warpers("tl_sample_proc", min_p, typical_p, epsilon, eta, &wp);
    if (rc != TL_OK) return rc;
    TL_REQUIRE(ws_bytes >= tl_logits_proc_ws(M, V), TL_ERR_WORKSPACE, "tl_sample_proc: workspace %zu < %zu", ws_bytes,
               tl_logits_proc_ws(M, V));
    cudaStream_t st = (cudaStream_t)stream;
    uint32_t* ban = (uint32_t*)workspace;
    const LpRows h{log, len, bits, (flags & TL_LP_BAN) ? ban : nullptr, params_dev, L, lp_words(V)};
    if (flags & TL_LP_BAN) {
        rc = lp_ban_launch(h, ban, M, V, st);
        if (rc != TL_OK) return rc;
    }
    u64* hist = (u64*)((unsigned char*)workspace + lp_ban_bytes(M, V));
    const float it = 1.0f / temperature;
    const bf16* x = (const bf16*)logits;
    const LogDesc l = lg ? *lg : LogDesc{};
    auto* k = lg ? (warpers_on(wp) ? sample_proc_kernel<true, true> : sample_proc_kernel<true, false>)
                 : (warpers_on(wp) ? sample_proc_kernel<false, true> : sample_proc_kernel<false, false>);
    k<<<M, SM_THREADS, 0, st>>>(x, ids_out, V, h, it, top_k, top_p, seed, counters_dev, hist, l, wp);
    return check_launch("tl_sample_proc");
}

int tl_sample_proc(const void* logits, int64_t* ids_out, int32_t* log, int32_t* len, uint32_t* bits,
                   const int32_t* params_dev, int flags, int M, int V, int L, float temperature, int top_k, float top_p,
                   unsigned long long seed, int32_t* counters_dev, void* workspace, size_t ws_bytes, void* stream, float min_p,
                   float typical_p, float epsilon, float eta) {
    return sample_proc_launch(logits, ids_out, log, len, bits, params_dev, flags, M, V, L, temperature, top_k, top_p, seed,
                              counters_dev, workspace, ws_bytes, nullptr, stream, min_p, typical_p, epsilon, eta);
}

int tl_sample_proc_log(const void* logits, int64_t* ids_out, int32_t* log, int32_t* len, uint32_t* bits,
                       const int32_t* params_dev, int flags, int M, int V, int L, float temperature, int top_k, float top_p,
                       unsigned long long seed, int32_t* counters_dev, void* workspace, size_t ws_bytes, float* raw_log,
                       float* score_log, int32_t* log_col, int n_cols, int B_total, int row0, void* stream, float min_p,
                       float typical_p, float epsilon, float eta) {
    using namespace tl;
    LogDesc lg;
    const int rc = make_log("tl_sample_proc_log", raw_log, score_log, log_col, n_cols, B_total, row0, M, V, temperature, &lg);
    if (rc != TL_OK) return rc;
    return sample_proc_launch(logits, ids_out, log, len, bits, params_dev, flags, M, V, L, temperature, top_k, top_p, seed,
                              counters_dev, workspace, ws_bytes, &lg, stream, min_p, typical_p, epsilon, eta);
}

size_t tl_sample_ws(int M) { return (size_t)(M > 0 ? M : 0) * tl::SM_BINS * sizeof(uint32_t); }

static int sample_launch(const void* logits, int64_t* ids_out, int M, int V, float temperature, int top_k, float top_p,
                         unsigned long long seed, int32_t* counters_dev, void* workspace, size_t ws_bytes, const tl::LogDesc* lg,
                         void* stream, float min_p, float typical_p, float epsilon, float eta) {
    using namespace tl;
    TL_REQUIRE(logits && ids_out && counters_dev && workspace, TL_ERR_INVALID, "tl_sample: null argument");
    TL_REQUIRE(M >= 1 && V >= 1, TL_ERR_INVALID, "tl_sample: bad shape M=%d V=%d", M, V);
    TL_REQUIRE(temperature > 0.f && top_p > 0.f && top_p <= 1.f && top_k >= 0, TL_ERR_INVALID,
               "tl_sample: temperature must be > 0, 0 < top_p <= 1, top_k >= 0 (got %g, %g, %d)", temperature, top_p, top_k);
    Warpers wp;
    const int rc = check_warpers("tl_sample", min_p, typical_p, epsilon, eta, &wp);
    if (rc != TL_OK) return rc;
    TL_REQUIRE(ws_bytes >= tl_sample_ws(M), TL_ERR_INVALID, "tl_sample: workspace too small");
    const LogDesc l = lg ? *lg : LogDesc{};
    auto* k = lg ? (warpers_on(wp) ? sample_kernel<true, true> : sample_kernel<true, false>)
                 : (warpers_on(wp) ? sample_kernel<false, true> : sample_kernel<false, false>);
    k<<<M, SM_THREADS, 0, (cudaStream_t)stream>>>((const bf16*)logits, ids_out, V, 1.0f / temperature, top_k, top_p, seed,
                                                 counters_dev, (uint32_t*)workspace, l, wp);
    return check_launch("tl_sample");
}

int tl_sample(const void* logits, int64_t* ids_out, int M, int V, float temperature, int top_k, float top_p,
              unsigned long long seed, int32_t* counters_dev, void* workspace, size_t ws_bytes, void* stream, float min_p,
              float typical_p, float epsilon, float eta) {
    return sample_launch(logits, ids_out, M, V, temperature, top_k, top_p, seed, counters_dev, workspace, ws_bytes, nullptr, stream,
                         min_p, typical_p, epsilon, eta);
}

int tl_sample_log(const void* logits, int64_t* ids_out, int M, int V, float temperature, int top_k, float top_p,
                  unsigned long long seed, int32_t* counters_dev, void* workspace, size_t ws_bytes, float* raw_log,
                  float* score_log, int32_t* log_col, int n_cols, int B_total, int row0, void* stream, float min_p, float typical_p,
                  float epsilon, float eta) {
    using namespace tl;
    LogDesc lg;
    const int rc = make_log("tl_sample_log", raw_log, score_log, log_col, n_cols, B_total, row0, M, V, temperature, &lg);
    if (rc != TL_OK) return rc;
    return sample_launch(logits, ids_out, M, V, temperature, top_k, top_p, seed, counters_dev, workspace, ws_bytes, &lg, stream,
                         min_p, typical_p, epsilon, eta);
}

size_t tl_spec_accept_ws(int K) {
    const size_t rows = (size_t)(K > 0 ? 2 * K + 1 : 0);
    return rows * tl::SM_BINS * sizeof(uint32_t) + rows * sizeof(tl::SpecRow);
}

int tl_spec_accept(const void* p_logits, int V_p, const void* q_logits, int V_q, int K, const int64_t* in_ids,
                   const int32_t* n_cand, float temperature, int top_k, float top_p, unsigned long long seed,
                   int32_t* counter_dev, int64_t* ids_out, void* workspace, size_t ws_bytes, void* stream, float min_p,
                   float typical_p, float epsilon, float eta) {
    using namespace tl;
    TL_REQUIRE(p_logits && q_logits && in_ids && n_cand && counter_dev && ids_out && workspace, TL_ERR_INVALID,
               "tl_spec_accept: null argument");
    TL_REQUIRE(K >= 1 && K <= TL_PL_MAX_DRAFT && V_p >= 1 && V_q >= 1, TL_ERR_INVALID,
               "tl_spec_accept: bad shape K=%d V_p=%d V_q=%d", K, V_p, V_q);
    TL_REQUIRE(temperature > 0.f && top_p > 0.f && top_p <= 1.f && top_k >= 0, TL_ERR_INVALID,
               "tl_spec_accept: temperature must be > 0, 0 < top_p <= 1, top_k >= 0 (got %g, %g, %d)", temperature, top_p, top_k);
    Warpers wp;
    int rc = check_warpers("tl_spec_accept", min_p, typical_p, epsilon, eta, &wp);
    if (rc != TL_OK) return rc;
    TL_REQUIRE(ws_bytes >= tl_spec_accept_ws(K), TL_ERR_INVALID, "tl_spec_accept: workspace %zu < %zu", ws_bytes,
               tl_spec_accept_ws(K));
    cudaStream_t st = (cudaStream_t)stream;
    uint32_t* hist = (uint32_t*)workspace;
    SpecRow* rows = (SpecRow*)(hist + (size_t)(2 * K + 1) * SM_BINS);
    const float inv_temp = 1.0f / temperature;
    const bool on = warpers_on(wp);
    (on ? spec_rows_kernel<true> : spec_rows_kernel<false>)<<<2 * K + 1, SM_THREADS, 0, st>>>(
        (const bf16*)p_logits, V_p, (const bf16*)q_logits, V_q, K, inv_temp, top_k, top_p, rows, hist, wp);
    rc = check_launch("tl_spec_accept");
    if (rc != TL_OK) return rc;
    (on ? spec_draw_kernel<true> : spec_draw_kernel<false>)<<<1, SM_THREADS, 0, st>>>(
        (const bf16*)p_logits, V_p, (const bf16*)q_logits, V_q, K, in_ids, n_cand, inv_temp, seed, counter_dev, rows, ids_out);
    return check_launch("tl_spec_accept");
}

}  // extern "C"
