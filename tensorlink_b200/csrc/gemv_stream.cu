// Decode-shaped Linear, v2: persistent weight-streaming GEMV with a bulk-copy (TMA) producer warp.
//
// One CTA per SM.  Work is handed out in units: P whole consecutive row PAIRS of W (pair = gate/up for the SwiGLU
// epilogue) when a pair fits one <= 16 KB ring stage, else one pair in K-chunks of one stage each.  Units are taken in
// address order from a ticket counter (common.cuh), so an SM that streams faster takes more of them, every CTA finishes
// within one ticket of the others, and the first units of a launch are the first bytes of W, which the previous launch
// asked L2 to prefetch.  Warp 8 is the producer: it takes tickets and issues cp.async.bulk copies of the units' stages
// into a deep shared-memory ring (mbarrier full/empty, ~190 KB in flight per SM), never waiting on the math, and
// records the unit of every stage beside the barriers.  Ring slot s is always drained by consumer warp s % NW, and a
// warp takes a whole unit (all of its K chunks, in order), so a dot product finishes with one warp reduction and no
// cross-warp traffic.  x (optionally RMS-normalised with HF rounding) is staged once per CTA while the producer is
// already streaming.
// Algorithmic bytes per launch = 2*N*K.
//
// The same kernel streams FP8 weights (WT = fp8_e4m3, tl_gemv_fp8): one byte per weight plus an fp32 scale per (row,
// 128-column group), read through L1.  Each weight is formed as bf16(float(w) * scale), the bf16 weight of HF's
// dequantized checkpoint, and every lane visits K in the bf16 kernel's order (lane v of a pass takes elements 8v..8v+7),
// so the FMA sequence of every output, and therefore the result, is the bf16 kernel's over the dequantized matrix.
// A stage then holds twice the rows, and a chunk of a chunked pair twice the columns.
#include <stdlib.h>

#include "common.cuh"
#include "fp8.cuh"

namespace tl {

constexpr int GS_CONSUMER_WARPS = 8;
constexpr int GS_THREADS = (GS_CONSUMER_WARPS + 1) * 32;
constexpr int GS_MAX_STAGES = 16;
constexpr int GS_STAGE_BYTES = 16 * 1024;
constexpr int GS_KC = 4096;            // K chunk (elements of a bf16 weight) when a pair does not fit one stage
constexpr int GS_SCALE_GROUP = 128;    // FP8 weights: one fp32 scale per row and 128 consecutive columns
// Bytes per ticket: one atomic round trip (~1 us under a full HBM stream) has to hide behind the ticket before it, and
// a CTA finishes at most one ticket after the others.
constexpr int GS_TICKET_BYTES = 24 * 1024;
constexpr int GS_SKIP = -2;            // s_unit: an empty stage the warp only hands back
constexpr int GS_LEAVE = -1;           // s_unit: no units left, the warp leaves

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// The body of both kernels below.  WT: bf16, or fp8_e4m3 with `scales` [N][K/128].
template <typename WT, int M>
__device__ __forceinline__ void
gemv_stream_body(const bf16* __restrict__ x, const WT* __restrict__ W, bf16* __restrict__ y, int N, int K,
                 const bf16* __restrict__ bias, const bf16* __restrict__ residual, const bf16* __restrict__ norm_w,
                 float eps, int flags, int P, int n_stages, int NW, int stage_bytes, int G, unsigned* __restrict__ ctr,
                 const unsigned char* __restrict__ pf_ptr, unsigned long long pf_bytes, const float* __restrict__ scales) {
    constexpr bool FP8 = sizeof(WT) == 1;
    constexpr int WB = sizeof(WT);                 // bytes per weight
    constexpr int KCW = GS_KC * 2 / WB;            // chunk columns: a chunk of a pair fills one 16 KB stage
    extern __shared__ __align__(128) unsigned char smem[];
    unsigned char* ring = smem;                                                    // [n_stages][stage_bytes]
    bf16* xs = reinterpret_cast<bf16*>(smem + (size_t)n_stages * stage_bytes);     // [M][K]
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + (size_t)n_stages * stage_bytes + (((size_t)M * K * 2 + 15) & ~(size_t)15));
    uint64_t* empty_bar = full_bar + GS_MAX_STAGES;
    __shared__ float s_part[GS_CONSUMER_WARPS][M];
    __shared__ int s_unit[GS_MAX_STAGES];      // unit in each ring slot (or GS_SKIP / GS_LEAVE), released by the full barrier

    // programmatic dependent launch: let the next kernel's CTAs start (and prefetch ITS weights) as SMs free up
    asm volatile("griddepcontrol.launch_dependents;");
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int npairs = N >> 1;
    const int n_units = (npairs + P - 1) / P;                          // unit = P consecutive pairs
    // NW consumer warps take units; n_stages %% NW == 0, so ring slot s is ALWAYS consumed by warp s %% NW and every
    // waiter observes every phase of the barriers it waits on (no mbarrier parity aliasing).
    const bool chunked = K > KCW || (size_t)K * (2 * WB) > GS_STAGE_BYTES;  // a pair does not fit one stage
    const int KC = chunked ? KCW : K;
    const int n_chunks = (K + KC - 1) / KC;

    if (tid == 0) {
        for (int s = 0; s < n_stages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 1);
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == GS_CONSUMER_WARPS) {
        // ================================================================= producer (one elected lane)
        if (lane == 0) {
            // CTA b's first ticket is units [b*G, (b+1)*G) without a round trip; later tickets come from the counter,
            // offset by the grid's first tickets.  The next ticket is requested while the current one is handed out.
            const int first = gridDim.x * G;
            const bool tickets = first < n_units;          // else the first tickets cover the matrix: no counter traffic
            int t_cur = blockIdx.x * G, t_used = 0;
            int t_next = tickets ? first + ticket_take(ctr, G) : n_units;
            auto next_unit = [&]() -> int {
                if (t_used == G) {
                    if (t_next >= n_units) return n_units;
                    t_cur = t_next;
                    t_used = 0;
                    t_next = first + ticket_take(ctr, G);
                }
                return t_cur + t_used++;
            };
            // per consumer warp: its unit and the next chunk of it.  A chunked unit takes n_chunks of the warp's
            // stages, so warp w first hands back w*n_chunks/NW empty stages: the warps then need new units at evenly
            // spread times instead of all at once, and a CTA never commits to NW units in one step.
            int unit[GS_CONSUMER_WARPS], chunk[GS_CONSUMER_WARPS], skip[GS_CONSUMER_WARPS];
#pragma unroll
            for (int w = 0; w < GS_CONSUMER_WARPS; ++w) {
                unit[w] = 0;
                chunk[w] = 0;
                skip[w] = chunked ? w * n_chunks / NW : 0;
            }
            int stage = 0, live = NW;
            uint32_t phase = 0;
            while (live > 0) {
#pragma unroll
                for (int w = 0; w < GS_CONSUMER_WARPS; ++w) {
                    if (w >= NW) continue;
                    if (unit[w] != GS_LEAVE) {          // the slots of a warp that left stay untouched
                        mbar_wait(&empty_bar[stage], phase ^ 1);
                        unsigned char* dst = ring + (size_t)stage * stage_bytes;
                        if (skip[w] > 0) {
                            --skip[w];
                            s_unit[stage] = GS_SKIP;
                            mbar_expect_tx(&full_bar[stage], 0);
                        } else {
                            if (chunk[w] == 0) {
                                unit[w] = next_unit();
                                if (unit[w] >= n_units) unit[w] = GS_LEAVE;
                            }
                            s_unit[stage] = unit[w];
                            if (unit[w] == GS_LEAVE) {
                                --live;
                                mbar_expect_tx(&full_bar[stage], 0);
                            } else if (!chunked) {   // np pairs = 2*np whole rows, contiguous in memory: one copy
                                const int pair0 = unit[w] * P;
                                const int np = min(P, npairs - pair0);
                                const uint32_t bytes = (uint32_t)(2 * np) * (uint32_t)K * (uint32_t)WB;
                                mbar_expect_tx(&full_bar[stage], bytes);
                                bulk_load_1d(dst, W + (size_t)(2 * pair0) * K, bytes, &full_bar[stage]);
                            } else {                 // one K chunk of the two rows of one pair: two copies
                                const int k0 = chunk[w] * KC;
                                const uint32_t bytes = (uint32_t)min(KC, K - k0) * (uint32_t)WB;
                                mbar_expect_tx(&full_bar[stage], 2 * bytes);
                                bulk_load_1d(dst, W + (size_t)(2 * unit[w]) * K + k0, bytes, &full_bar[stage]);
                                bulk_load_1d(dst + (size_t)KC * WB, W + (size_t)(2 * unit[w] + 1) * K + k0, bytes, &full_bar[stage]);
                                if (++chunk[w] == n_chunks) chunk[w] = 0;
                            }
                        }
                    }
                    if (++stage == n_stages) { stage = 0; phase ^= 1; }
                }
            }
            // this CTA takes no more tickets: the last CTA out zeroes the counter for the next launch on these words
            if (tickets && last_cta_out(ctr + 1)) {
                ctr[0] = 0u;
                __threadfence();
            }
            // every load of this CTA is issued (the last ring-full is still in flight): queue L2 prefetches of this
            // CTA's slice of the NEXT kernel's weights behind them, so HBM keeps streaming through this kernel's tail,
            // the launch boundary and the next kernel's prologue; the next kernel then fills its ring from L2.
            if (pf_bytes) {
                const unsigned long long per = ((pf_bytes / gridDim.x) + 4095ull) & ~4095ull;
                unsigned long long off = (unsigned long long)blockIdx.x * per;
                const unsigned long long end = off + per < pf_bytes ? off + per : pf_bytes;
                for (; off < end; off += 16384ull) {
                    const uint32_t sz = (uint32_t)(end - off < 16384ull ? end - off : 16384ull);
                    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(pf_ptr + off), "r"(sz) : "memory");
                }
            }
        }
    } else {
        // ================================================================= consumers
        // x / residual are produced by the previous kernel: wait for it (no-op without the PDL launch attribute);
        // the producer warp above streams weights, which nobody writes, without waiting.
        asm volatile("griddepcontrol.wait;" ::: "memory");
        const int nvec = K >> 3;
        if (norm_w) {
            float ss[M];
#pragma unroll
            for (int m = 0; m < M; ++m) ss[m] = 0.f;
            for (int v = tid; v < nvec; v += GS_CONSUMER_WARPS * 32) {
#pragma unroll
                for (int m = 0; m < M; ++m) {
                    const uint4 u = reinterpret_cast<const uint4*>(x + (size_t)m * K)[v];
                    const uint32_t* u32 = reinterpret_cast<const uint32_t*>(&u);
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const float a = bf16_lo(u32[j]), b = bf16_hi(u32[j]);
                        ss[m] += a * a + b * b;
                    }
                }
            }
#pragma unroll
            for (int m = 0; m < M; ++m) {
                const float t = warp_sum(ss[m]);
                if (lane == 0) s_part[warp][m] = t;
            }
            named_bar_sync(1, GS_CONSUMER_WARPS * 32);
            float rstd[M];
#pragma unroll
            for (int m = 0; m < M; ++m) {
                float t = 0.f;
#pragma unroll
                for (int w = 0; w < GS_CONSUMER_WARPS; ++w) t += s_part[w][m];
                rstd[m] = 1.0f / sqrtf(t / (float)K + eps);
            }
            for (int v = tid; v < nvec; v += GS_CONSUMER_WARPS * 32) {
                const uint4 g = reinterpret_cast<const uint4*>(norm_w)[v];
                const uint32_t* g32 = reinterpret_cast<const uint32_t*>(&g);
#pragma unroll
                for (int m = 0; m < M; ++m) {
                    const uint4 u = reinterpret_cast<const uint4*>(x + (size_t)m * K)[v];
                    uint4 o;
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
            for (int v = tid; v < nvec * M; v += GS_CONSUMER_WARPS * 32)
                reinterpret_cast<uint4*>(xs)[v] = reinterpret_cast<const uint4*>(x)[v];
        }
        named_bar_sync(1, GS_CONSUMER_WARPS * 32);

        const bool swiglu = flags & TL_EPI_SWIGLU;
        const int n_out = swiglu ? npairs : N;
        // epilogue for one finished pair (all lanes hold the reduced sums)
        auto finish = [&](int pair, const float (&a0)[M], const float (&a1)[M]) {
            if (lane != 0) return;
            const int r0 = 2 * pair;
#pragma unroll
            for (int m = 0; m < M; ++m) {
                float v0 = a0[m], v1 = a1[m];
                if (flags & TL_EPI_BIAS) {
                    v0 += bf2f(bias[r0]);
                    v1 += bf2f(bias[r0 + 1]);
                }
                if (swiglu) {
                    const float gate = rbf(v0), up = rbf(v1);
                    y[(size_t)m * n_out + pair] = f2bf(rbf(silu_f(gate)) * up);
                } else {
                    float t0 = rbf(v0), t1 = rbf(v1);
                    if (flags & TL_EPI_RESIDUAL) {
                        t0 += bf2f(residual[(size_t)m * N + r0]);
                        t1 += bf2f(residual[(size_t)m * N + r0 + 1]);
                    }
                    *reinterpret_cast<uint32_t*>(y + (size_t)m * N + r0) = pack_bf16(t0, t1);
                }
            }
        };
        // dot product of `vecs` 8-weight vectors of two rows (stage rows r0, r1 = W rows row0, row0 + 1) against x[k0..]
        auto dot2 = [&](const unsigned char* r0, const unsigned char* r1, int row0, int k0, int vecs, float (&a0)[M],
                        float (&a1)[M]) {
          if constexpr (FP8) {
            const int n_groups = K / GS_SCALE_GROUP;
            const float* s0 = scales + (size_t)row0 * n_groups + k0 / GS_SCALE_GROUP;
            const float* s1 = s0 + n_groups;
#pragma unroll 4
            for (int v = lane; v < vecs; v += 32) {
                float w0[8], w1[8];
                fp8x8_scaled(reinterpret_cast<const uint2*>(r0)[v], __ldg(s0 + (v >> 4)), w0);
                fp8x8_scaled(reinterpret_cast<const uint2*>(r1)[v], __ldg(s1 + (v >> 4)), w1);
#pragma unroll
                for (int m = 0; m < M; ++m) {
                    const uint4 xv = reinterpret_cast<const uint4*>(xs + (size_t)m * K + k0)[v];
                    const uint32_t* x32 = reinterpret_cast<const uint32_t*>(&xv);
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const float xl = bf16_lo(x32[j]), xh = bf16_hi(x32[j]);
                        a0[m] = fmaf(w0[2 * j], xl, a0[m]);
                        a0[m] = fmaf(w0[2 * j + 1], xh, a0[m]);
                        a1[m] = fmaf(w1[2 * j], xl, a1[m]);
                        a1[m] = fmaf(w1[2 * j + 1], xh, a1[m]);
                    }
                }
            }
          } else {
#pragma unroll 4
            for (int v = lane; v < vecs; v += 32) {
                const uint4 w0 = reinterpret_cast<const uint4*>(r0)[v], w1 = reinterpret_cast<const uint4*>(r1)[v];
                const uint32_t* a32 = reinterpret_cast<const uint32_t*>(&w0);
                const uint32_t* b32 = reinterpret_cast<const uint32_t*>(&w1);
#pragma unroll
                for (int m = 0; m < M; ++m) {
                    const uint4 xv = reinterpret_cast<const uint4*>(xs + (size_t)m * K + k0)[v];
                    const uint32_t* x32 = reinterpret_cast<const uint32_t*>(&xv);
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const float xl = bf16_lo(x32[j]), xh = bf16_hi(x32[j]);
                        a0[m] = fmaf(bf16_lo(a32[j]), xl, a0[m]);
                        a0[m] = fmaf(bf16_hi(a32[j]), xh, a0[m]);
                        a1[m] = fmaf(bf16_lo(b32[j]), xl, a1[m]);
                        a1[m] = fmaf(bf16_hi(b32[j]), xh, a1[m]);
                    }
                }
            }
          }
        };
        // this warp's stages are sequence numbers warp, warp+NW, warp+2*NW, ... of the producer's order; the producer
        // says in s_unit which unit each one holds
        int seq = warp, c = 0;
        float a0[M], a1[M];
#pragma unroll
        for (int m = 0; m < M; ++m) a0[m] = a1[m] = 0.f;
        while (warp < NW) {
            const int stage = seq % n_stages;
            const uint32_t phase = (uint32_t)(seq / n_stages) & 1u;
            mbar_wait(&full_bar[stage], phase);
            const int unit = s_unit[stage];
            if (unit == GS_LEAVE) break;
            const unsigned char* src = ring + (size_t)stage * stage_bytes;
            if (unit >= 0 && !chunked) {
                const int pair0 = unit * P;
                const int np = min(P, npairs - pair0);
                for (int pp = 0; pp < np; ++pp) {
                    float b0[M], b1[M];
#pragma unroll
                    for (int m = 0; m < M; ++m) b0[m] = b1[m] = 0.f;
                    dot2(src + (size_t)(2 * pp) * K * WB, src + (size_t)(2 * pp + 1) * K * WB, 2 * (pair0 + pp), 0, nvec,
                         b0, b1);
#pragma unroll
                    for (int m = 0; m < M; ++m) { b0[m] = warp_sum(b0[m]); b1[m] = warp_sum(b1[m]); }
                    finish(pair0 + pp, b0, b1);
                }
            } else if (unit >= 0) {
                const int k0 = c * KC;
                dot2(src, src + (size_t)KC * WB, 2 * unit, k0, min(KC, K - k0) >> 3, a0, a1);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[stage]);
            seq += NW;
            if (unit >= 0 && chunked && ++c == n_chunks) {     // the unit's last chunk: the pair is done
#pragma unroll
                for (int m = 0; m < M; ++m) { a0[m] = warp_sum(a0[m]); a1[m] = warp_sum(a1[m]); }
                finish(unit, a0, a1);
#pragma unroll
                for (int m = 0; m < M; ++m) a0[m] = a1[m] = 0.f;
                c = 0;
            }
        }
    }
}

template <int M>
__global__ void __launch_bounds__(GS_THREADS, 1)
gemv_stream_kernel(const bf16* __restrict__ x, const bf16* __restrict__ W, bf16* __restrict__ y, int N, int K,
                   const bf16* __restrict__ bias, const bf16* __restrict__ residual, const bf16* __restrict__ norm_w,
                   float eps, int flags, int P, int n_stages, int NW, int stage_bytes, int G, unsigned* __restrict__ ctr,
                   const unsigned char* __restrict__ pf_ptr, unsigned long long pf_bytes) {
    gemv_stream_body<bf16, M>(x, W, y, N, K, bias, residual, norm_w, eps, flags, P, n_stages, NW, stage_bytes, G, ctr,
                              pf_ptr, pf_bytes, nullptr);
}

template <int M>
__global__ void __launch_bounds__(GS_THREADS, 1)
gemv_stream_fp8_kernel(const bf16* __restrict__ x, const fp8_e4m3* __restrict__ W, bf16* __restrict__ y, int N, int K,
                       const bf16* __restrict__ bias, const bf16* __restrict__ residual, const bf16* __restrict__ norm_w,
                       float eps, int flags, int P, int n_stages, int NW, int stage_bytes, int G,
                       unsigned* __restrict__ ctr, const unsigned char* __restrict__ pf_ptr, unsigned long long pf_bytes,
                       const float* __restrict__ scales) {
    gemv_stream_body<fp8_e4m3, M>(x, W, y, N, K, bias, residual, norm_w, eps, flags, P, n_stages, NW, stage_bytes, G,
                                  ctr, pf_ptr, pf_bytes, scales);
}

template <typename WT, int M>
static int launch_stream(const void* x, const void* W, const float* scales, void* y, int N, int K, const void* bias,
                         const void* residual, const void* norm_w, float eps, int flags, unsigned* ctr, const void* pf_ptr,
                         size_t pf_bytes, cudaStream_t st) {
    constexpr size_t WB = sizeof(WT);
    const char* what = WB == 1 ? "tl_gemv_fp8/stream" : "tl_gemv_bf16/stream";
    constexpr bool FP8 = WB == 1;
    void* kern = FP8 ? (void*)gemv_stream_fp8_kernel<M> : (void*)gemv_stream_kernel<M>;
    // Two half-size rings per SM (16 consumer warps, finer work split, the next kernel's CTAs become resident as soon as
    // one of the two exits) when an SM's share of W is small — the latency-bound regime of small models; one deep
    // ring per SM otherwise.  The 128 KB threshold has not been re-chosen by measurement on H100.
    // TL_GEMV_CTAS_PER_SM=1|2 forces either.
    static int forced = -1;
    if (forced < 0) {
        const char* e = getenv("TL_GEMV_CTAS_PER_SM");
        forced = (e && e[0] == '2') ? 2 : ((e && e[0] == '1') ? 1 : 0);
    }
    int per_sm = forced ? forced : (((size_t)N * K * WB / (size_t)sm_count() <= (size_t)128 * 1024) ? 2 : 1);
    // TL_GEMV_RING_KB (default 220): shared memory per CTA.  <= 110 leaves room for the NEXT kernel's CTA on the same
    // SM, so under programmatic dependent launch its producer fills its ring while this kernel is still streaming.
    static int ring_kb = 0;
    if (ring_kb == 0) {
        const char* e = getenv("TL_GEMV_RING_KB");
        ring_kb = e ? atoi(e) : 220;
        if (ring_kb < 48 || ring_kb > 220) ring_kb = 220;
    }
    const size_t xs_bytes = (((size_t)M * K * 2) + 15) & ~(size_t)15;
    const size_t fixed = xs_bytes + 2 * GS_MAX_STAGES * sizeof(uint64_t);
    if constexpr (FP8) {
        // The FP8 kernel runs exactly where the bf16 kernel would run on this shape, and the register-streaming
        // fallback everywhere else, so an FP8 GEMV takes the kernel (and the summation order) of the bf16 GEMV over the
        // dequantized weights.  Its own ring then takes one CTA per SM when two half-size rings would be too shallow.
        auto stages = [&](int wb, int ps) -> int64_t {
            const bool ch = K > GS_KC * 2 / wb || (size_t)K * 2 * wb > GS_STAGE_BYTES;
            int p = ch ? 1 : (int)(GS_STAGE_BYTES / ((size_t)K * 2 * wb));
            p = p < 1 ? 1 : (p > 8 ? 8 : p);
            const int64_t sb = ch ? GS_STAGE_BYTES : (int64_t)((((size_t)p * K * 2 * wb) + 127) & ~(size_t)127);
            return ((int64_t)(ps == 2 ? 110 * 1024 : ring_kb * 1024) - (int64_t)fixed) / sb;
        };
        const int per_sm_bf16 = forced ? forced : (((size_t)N * K * 2 / (size_t)sm_count() <= (size_t)128 * 1024) ? 2 : 1);
        if (stages(2, per_sm_bf16) < 4) return 1;
        if (per_sm == 2 && stages(1, 2) < 4) per_sm = 1;
    }
    const int SMEM_CAP = per_sm == 2 ? 110 * 1024 : ring_kb * 1024;
    static bool attr_done = false;
    if (!attr_done) {
        if (cudaFuncSetAttribute((const void*)kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024) != cudaSuccess)
            return check_launch(what);
        attr_done = true;
    }
    const int KCW = GS_KC * 2 / (int)WB;
    const bool chunked = K > KCW || (size_t)K * 2 * WB > GS_STAGE_BYTES;
    int P = chunked ? 1 : (int)(GS_STAGE_BYTES / ((size_t)K * 2 * WB));
    if (P < 1) P = 1;
    if (P > 8) P = 8;
    // a stage holds one unit: up to P whole pairs, or one 16 KB chunk of one pair
    const int stage_bytes = chunked ? GS_STAGE_BYTES : (int)((((size_t)P * K * 2 * WB) + 127) & ~(size_t)127);
    int max_stages = (int)((SMEM_CAP - fixed) / stage_bytes);
    if (max_stages > GS_MAX_STAGES) max_stages = GS_MAX_STAGES;
    if (max_stages < 4) return 1;   // caller falls back to the register-streaming kernel
    // pick (n_stages, NW): n_stages a multiple of NW, as many bytes in flight as possible, then as many warps
    int n_stages = 0, NW = 0;
    for (int nw = GS_CONSUMER_WARPS; nw >= 4; --nw) {
        const int st_ = max_stages / nw * nw;
        if (st_ > n_stages) { n_stages = st_; NW = nw; }
    }
    const size_t smem = (size_t)n_stages * stage_bytes + fixed;
    const int npairs = N >> 1;
    int grid = sm_count() * per_sm;
    if (grid > npairs) grid = npairs;
    // Few pairs per CTA (the latency-bound launches of small models): one pair per unit and every CTA's first ticket
    // covers its share, so no CTA waits for a ticket round trip; the split is then as even as a static one.
    int G;
    if (npairs <= 8 * grid) {
        P = 1;
        G = (npairs + grid - 1) / grid;
    } else {
        const int unit_bytes = (int)(chunked ? K * 2 * WB : P * K * 2 * WB);
        G = (GS_TICKET_BYTES + unit_bytes - 1) / unit_bytes;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(GS_THREADS);
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
    if constexpr (FP8)
        cudaLaunchKernelEx(&cfg, gemv_stream_fp8_kernel<M>, (const bf16*)x, (const fp8_e4m3*)W, (bf16*)y, N, K,
                           (const bf16*)bias, (const bf16*)residual, (const bf16*)norm_w, eps, flags, P, n_stages, NW,
                           stage_bytes, G, ctr, (const unsigned char*)pf_ptr, (unsigned long long)(pf_bytes & ~(size_t)15),
                           scales);
    else
        cudaLaunchKernelEx(&cfg, gemv_stream_kernel<M>, (const bf16*)x, (const bf16*)W, (bf16*)y, N, K, (const bf16*)bias,
                           (const bf16*)residual, (const bf16*)norm_w, eps, flags, P, n_stages, NW, stage_bytes, G, ctr,
                           (const unsigned char*)pf_ptr, (unsigned long long)(pf_bytes & ~(size_t)15));
    return check_launch(what);
}

template <typename WT>
static int stream_dispatch(const void* x, const void* W, const float* scales, void* y, int M, int N, int K,
                           const void* bias, const void* residual, const void* norm_w, float eps, int flags, unsigned* ctr,
                           const void* pf_ptr, size_t pf_bytes, cudaStream_t st) {
    if (K % 8 != 0 || ((uintptr_t)W & 15)) return 1;
    if ((uintptr_t)pf_ptr & 15) pf_bytes = 0;
    switch (M) {
        case 1: return launch_stream<WT, 1>(x, W, scales, y, N, K, bias, residual, norm_w, eps, flags, ctr, pf_ptr, pf_bytes, st);
        case 2: return launch_stream<WT, 2>(x, W, scales, y, N, K, bias, residual, norm_w, eps, flags, ctr, pf_ptr, pf_bytes, st);
        case 3: return launch_stream<WT, 3>(x, W, scales, y, N, K, bias, residual, norm_w, eps, flags, ctr, pf_ptr, pf_bytes, st);
        case 4: return launch_stream<WT, 4>(x, W, scales, y, N, K, bias, residual, norm_w, eps, flags, ctr, pf_ptr, pf_bytes, st);
        default: return 1;
    }
}

// returns TL_OK, an error, or 1 = "not applicable, use the fallback kernel"
int gemv_stream_dispatch(const void* x, const void* W, void* y, int M, int N, int K, const void* bias,
                         const void* residual, const void* norm_w, float eps, int flags, unsigned* ctr, const void* pf_ptr,
                         size_t pf_bytes, cudaStream_t st) {
    return stream_dispatch<bf16>(x, W, nullptr, y, M, N, K, bias, residual, norm_w, eps, flags, ctr, pf_ptr, pf_bytes, st);
}

// FP8 weights (scales [N][K/128] fp32): TL_OK, an error, or 1 = "the shapes do not fit the stream kernel"
int gemv_stream_fp8_dispatch(const void* x, const void* W, const float* scales, void* y, int M, int N, int K,
                             const void* bias, const void* residual, const void* norm_w, float eps, int flags, unsigned* ctr,
                             const void* pf_ptr, size_t pf_bytes, cudaStream_t st) {
    return stream_dispatch<fp8_e4m3>(x, W, scales, y, M, N, K, bias, residual, norm_w, eps, flags, ctr, pf_ptr, pf_bytes,
                                     st);
}

}  // namespace tl
