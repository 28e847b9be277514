// A chain of dependent decode-step jobs as ONE persistent kernel: the HBM stream never stops at a dependency.
//
// The per-kernel decode path (gemv_stream.cu + attention.cu) pays, at every launch boundary, the tail of one kernel,
// the ramp-up of the next and (for the attention launch) a few microseconds in which nothing streams at all: the two
// small Linears of a layer (qkv 33 MB, o 26 MB at Qwen2.5-7B) lose the most to that.
// Here one CTA per SM stays resident for a whole decoder layer (or any job list up to DC_MAX_JOBS) and walks it:
//
//     ATTN(j)  ->  GEMV o(j) (+residual)  ->  GEMV gate/up(j) (+norm, SwiGLU)  ->  GEMV down(j) (+residual)
//              ->  GEMV qkv(j+1) (+norm, bias)
//
// * The producer warp streams the weight rows of EVERY GEMV job of the chain, in order, into one shared-memory ring
//   (cp.async.bulk, mbarrier full/empty) and never waits for a dependency: weights are constant.  While the consumer
//   warps cross a grid barrier, stage the next input vector or run the attention job, the ring (~160-190 KB per SM)
//   fills with the next job's weights.
// * A dependency is one counter in global memory: writers publish with red.release.gpu, every CTA's thread 0 polls
//   with ld.acquire.gpu.  No cooperative-groups grid sync, no per-thread fences.  Every spin gives up after 2 s and
//   raises an error word instead of hanging the GPU.
// * Units of a GEMV job (one ring stage of consecutive weight rows) are handed out in groups by a ticket counter, not
//   split statically: an SM that streams faster takes more groups, so all CTAs finish a job within one group of each
//   other and the dependency wait behind it stays shorter than what the ring bridges.
// * The attention job is split-KV over ALL CTAs, once per kv head (GQA: the n_rep query heads that share a kv head are
//   handled together, so every cached key / value byte is read exactly once chip-wide): CTA = (row, kv head, key
//   range); inside it warp r owns query head r end to end over 32-key tiles staged in shared memory (scores with
//   lane = key, online softmax in registers, P.V with lane = output dims; the tile's global loads fly under the q
//   round trip) -> partial (m, l, o) per query head -> the last CTA of a group to arrive combines the partials and
//   publishes the group; RoPE, the Qwen3 q/k norm and the KV append are fused in.
// * Job descriptors travel in kernel parameter space (constant bank): no global-memory fetch at a job boundary.
// * Programmatic dependent launch on both sides; after its last load the producer queues L2 prefetches of the next
//   launch's first weights.
// Arithmetic and rounding points of the GEMV jobs are those of gemv_stream_kernel (bit-identical); the attention
// job follows the SDPA contract of attn_decode_* (P rounded to bf16 before P.V, fp32 accumulation).
// Algorithmic bytes per launch = sum over the GEMV jobs of 2*N*K  +  the KV bytes of the attention jobs.
#include <stdlib.h>

#include "common.cuh"

namespace tl {

constexpr int DC_CW = 8;                       // consumer warps
constexpr int DC_CT = DC_CW * 32;              // consumer threads
constexpr int DC_THREADS = DC_CT + 32;         // + producer warp
constexpr int DC_MAX_STAGES = 24;
constexpr int DC_MAX_JOBS = 16;
constexpr int DC_MAX_M = 4;
constexpr int DC_TILE = 32;                    // keys per attention tile (an attention CTA takes whole tiles)
constexpr int DC_MIN_KEYS = 128;               // ... and at least this many keys: contexts up to here need no partials / combine
constexpr int DC_KT_MAX = 128 * 2 + 16;        // bytes per K / V tile row at d = 128 (16 bytes of padding: conflict-free rows)
// shared memory of the attention job: sq[8][128] f32 | sk[128] sv[128] f32 | sp[8][32] f32 | K tile | V tile
constexpr int DC_ATTN_BYTES = 8 * 128 * 4 + 2 * 128 * 4 + 8 * DC_TILE * 4 + 2 * DC_TILE * DC_KT_MAX;
constexpr int DC_GB = 8;                       // ring of unit-group tickets (> n_stages / NW + 1: the producer's lead in groups)
constexpr int DC_JOBCTR = 64;                  // word offset of the per-job unit counters inside a sync slot
constexpr int DC_STAT_OFF = 2 * (DC_MAX_JOBS + 1) * 4 + DC_MAX_JOBS * 160;   // trace: per-job wait / busy cycle counters
constexpr unsigned long long DC_TIMEOUT_NS = 2000000000ull;

struct ChainParams {
    int n_jobs, n_stages, NW, xs_bytes;
    int dynamic, stage_bytes;       // dynamic: units are handed out by tickets (1) or split statically per CTA (0)
    int kc, l2_ahead;               // stage_bytes: one ring slot; kc: K chunk (elements) of a row pair that exceeds a slot;
                                    // l2_ahead: bytes per CTA the L2 prefetch cursor may lead the shared-memory loads by
    unsigned* sync;                 // [0] barrier, [1] exit, [2] error, [4..] attention group counters, [64..] unit tickets
    float* attn_part;               // [M*n_h][cpg][D+4] partial (o[D], m, l, pad, pad)
    const unsigned char* pf_ptr;
    unsigned long long pf_bytes;
    unsigned long long* trace;      // optional (tools/trace_chain.py): globaltimer stamps of CTA 0 and the last CTA
    tl_decode_job jobs[DC_MAX_JOBS];
};

__device__ __forceinline__ void dc_bar(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ unsigned dc_ld_acquire(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void dc_red_release(unsigned* p, unsigned v) {
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long dc_timer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ uint4 dc_ldcg_v4(const void* p) {      // L2-coherent load of data written by other CTAs
    uint4 r;
    asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ float dc_ldcg_bf16(const bf16* p) {
    unsigned short v;
    asm volatile("ld.global.cg.u16 %0, [%1];" : "=h"(v) : "l"(p));
    return __uint_as_float(((uint32_t)v) << 16);
}
// wait on an mbarrier, giving up when the CTA has been declared dead (a grid-level wait timed out)
__device__ __forceinline__ bool dc_mbar_wait(uint64_t* bar, uint32_t parity, volatile int* dead) {
    int it = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (((++it) & 0xfff) == 0 && *dead) return false;
    }
    return true;
}

// A unit = P consecutive row pairs (one ring stage when a pair fits) or one pair in n_chunks K-chunks (one stage each).
// Units are numbered over the whole matrix.  Static mode: CTA c owns the contiguous units [u_begin, u_end).  Dynamic mode:
// groups of NW consecutive units are handed out by a ticket counter, so a faster SM simply takes more groups and every
// CTA finishes a job within one group of the others.
struct DcGeom {
    int npairs, P, U, u_begin, u_end, KC, n_chunks;
    bool chunked;
};
__device__ __forceinline__ DcGeom dc_geom(int N, int K, int DC_STAGE, int DC_KC) {
    DcGeom g;
    g.npairs = N >> 1;
    g.chunked = K > DC_KC || (size_t)K * 4 > (size_t)DC_STAGE;
    g.P = g.chunked ? 1 : min(8, (int)(DC_STAGE / ((size_t)K * 4)));
    g.U = (g.npairs + g.P - 1) / g.P;
    g.u_begin = (int)((long long)blockIdx.x * g.U / gridDim.x);
    g.u_end = (int)((long long)(blockIdx.x + 1) * g.U / gridDim.x);
    g.KC = g.chunked ? DC_KC : K;
    g.n_chunks = (K + g.KC - 1) / g.KC;
    return g;
}

template <int M>
__global__ void __launch_bounds__(DC_THREADS, 1) decode_chain_kernel(const __grid_constant__ ChainParams p) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int n_stages = p.n_stages, NW = p.NW, DC_STAGE = p.stage_bytes, DC_KC = p.kc;
    unsigned char* ring = smem;
    bf16* xs = reinterpret_cast<bf16*>(smem + (size_t)n_stages * DC_STAGE);                       // [M][K_max]
    unsigned char* attn_s = smem + (size_t)n_stages * DC_STAGE + (size_t)p.xs_bytes;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(attn_s + DC_ATTN_BYTES);
    uint64_t* empty_bar = full_bar + DC_MAX_STAGES;
    __shared__ float s_part[DC_CW][M];
    __shared__ int s_dead, s_last;
    __shared__ int s_gbase[DC_GB];            // first unit of the unit groups in flight (written by the producer)

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) {
        for (int s = 0; s < n_stages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 1);
        }
        s_dead = 0;
        s_last = 0;
        fence_barrier_init();
    }
    __syncthreads();
    // programmatic dependent launch: the next kernel may be scheduled as soon as every CTA of this grid is past this
    // point (its CTAs become resident as ours exit; its producer then streams while our last CTAs drain)
    asm volatile("griddepcontrol.launch_dependents;");

    if (warp == DC_CW) {
        // ================================================================= producer: weights of every GEMV job, in order
        if (lane == 0) {
            int stage = 0, gseq = 0;
            uint32_t phase = 0;
            bool alive = true;
            unsigned* const tickets = p.sync + DC_JOBCTR;
            // Second-level ring (static split only): an L2 prefetch cursor runs over this CTA's weight ranges of all jobs,
            // up to l2_ahead bytes in front of the shared-memory loads.  When the ring is full (consumers are crossing a
            // dependency) the producer keeps HBM streaming into L2; afterwards the ring refills at L2 speed.
            long long loaded = 0, prefetched = 0;
            int pf_job = 0;
            long long pf_off = 0;
            auto pf_range = [&](int j, const unsigned char*& base, long long& len) {
                const tl_decode_job& q = p.jobs[j];
                const DcGeom h = dc_geom(q.N, q.K, DC_STAGE, DC_KC);
                const long long r0 = (long long)h.u_begin * h.P * 2, r1 = min((long long)h.u_end * h.P * 2, (long long)q.N);
                base = reinterpret_cast<const unsigned char*>(q.W) + r0 * q.K * 2;
                len = (r1 - r0) * q.K * 2;
            };
            auto pump = [&](int max_issue) {
                if (p.dynamic || p.l2_ahead <= 0) return;
                while (max_issue-- > 0 && pf_job < p.n_jobs && prefetched < loaded + p.l2_ahead) {
                    if (p.jobs[pf_job].type != TL_JOB_GEMV) { ++pf_job; pf_off = 0; continue; }
                    const unsigned char* base;
                    long long len;
                    pf_range(pf_job, base, len);
                    if (pf_off >= len) { ++pf_job; pf_off = 0; continue; }
                    const uint32_t sz = (uint32_t)min(16384ll, len - pf_off);
                    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(base + pf_off), "r"(sz & ~15u) : "memory");
                    pf_off += sz;
                    prefetched += sz;
                }
            };
            // the first ticket of a job is requested one job ahead: its round trip never stalls the stream
            int first_ticket = 0;
            int jn = 0;
            while (jn < p.n_jobs && p.jobs[jn].type != TL_JOB_GEMV) ++jn;
            if (p.dynamic && jn < p.n_jobs) first_ticket = ticket_take(&tickets[jn], NW);
            for (int j = jn; j < p.n_jobs && alive; j = jn) {
                const tl_decode_job& jb = p.jobs[j];
                jn = j + 1;
                while (jn < p.n_jobs && p.jobs[jn].type != TL_JOB_GEMV) ++jn;
                const DcGeom g = dc_geom(jb.N, jb.K, DC_STAGE, DC_KC);
                const bf16* W = reinterpret_cast<const bf16*>(jb.W);
                const int K = jb.K;
                int base = p.dynamic ? first_ticket : g.u_begin;
                const int u_end = p.dynamic ? g.U : g.u_end;
                long long pwait = 0;
                if (p.dynamic && jn < p.n_jobs) first_ticket = ticket_take(&tickets[jn], NW);
                for (;;) {
                    const bool term = base >= u_end;                 // terminator group: NW empty stages, consumers leave the job
                    int next = base + NW;
                    if (p.dynamic && !term) next = ticket_take(&tickets[j], NW);   // used one group later
                    const int n_c = term ? 1 : g.n_chunks;
                    for (int c = 0; c < n_c && alive; ++c)
                        for (int w = 0; w < NW; ++w) {
                            const int unit = base + w;
                            const long long tw0 = clock64();
                            pump(2);
                            {
                                int it = 0;
                                while (!mbar_try_wait(&empty_bar[stage], phase ^ 1)) {      // ring full: keep HBM busy through L2
                                    pump(1);
                                    if (((++it) & 0xfff) == 0 && s_dead) { alive = false; break; }
                                }
                                if (!alive) break;
                            }
                            pwait += clock64() - tw0;
                            if (c == 0 && w == 0) s_gbase[gseq & (DC_GB - 1)] = term ? -1 : base;   // (released by the arrive below)
                            unsigned char* dst = ring + (size_t)stage * DC_STAGE;
                            if (term || unit >= u_end) {
                                mbar_expect_tx(&full_bar[stage], 0);
                            } else {
                                const int pair0 = unit * g.P;
                                const int np = min(g.P, g.npairs - pair0);
                                if (!g.chunked) {
                                    const uint32_t bytes = (uint32_t)(2 * np) * (uint32_t)K * 2u;
                                    mbar_expect_tx(&full_bar[stage], bytes);
                                    bulk_load_1d(dst, W + (size_t)(2 * pair0) * K, bytes, &full_bar[stage]);
                                    loaded += bytes;
                                } else {
                                    const int k0 = c * g.KC;
                                    const uint32_t bytes = (uint32_t)min(g.KC, K - k0) * 2u;
                                    mbar_expect_tx(&full_bar[stage], 2 * bytes);
                                    bulk_load_1d(dst, W + (size_t)(2 * pair0) * K + k0, bytes, &full_bar[stage]);
                                    bulk_load_1d(dst + (size_t)g.KC * 2, W + (size_t)(2 * pair0 + 1) * K + k0, bytes, &full_bar[stage]);
                                    loaded += 2 * bytes;
                                }
                            }
                            if (++stage == n_stages) { stage = 0; phase ^= 1; }
                        }
                    ++gseq;
                    if (term || !alive) break;
                    base = next;
                }
                if (p.trace && blockIdx.x == 0) p.trace[DC_STAT_OFF + (size_t)j * 4 + 2] = (unsigned long long)pwait;
            }
            // every load of this CTA is issued: queue L2 prefetches of this CTA's slice of the NEXT launch's first weights
            if (alive && p.pf_bytes) {
                const unsigned long long per = ((p.pf_bytes / gridDim.x) + 4095ull) & ~4095ull;
                unsigned long long off = (unsigned long long)blockIdx.x * per;
                const unsigned long long end = off + per < p.pf_bytes ? off + per : p.pf_bytes;
                for (; off < end; off += 16384ull) {
                    const uint32_t sz = (uint32_t)(end - off < 16384ull ? end - off : 16384ull);
                    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p.pf_ptr + off), "r"(sz) : "memory");
                }
            }
        }
        return;
    }

    // ===================================================================== consumers (256 threads)
    unsigned* const bar_ctr = p.sync;
    unsigned* const err_word = p.sync + 2;
    unsigned* const grp_ctr = p.sync + 4;
    unsigned bar_target = 0;
    // One dependency: `n_arrivals` publishers (this CTA is one of them iff `arrive`), every CTA waits for all of them.
    // Returns false when the wait timed out (the CTA then leaves the job loop; the host sees the error word).
    auto grid_dep = [&](bool arrive, unsigned n_arrivals) -> bool {
        dc_bar(1, DC_CT);                              // every consumer thread's stores of this job are issued
        if (tid == 0) {
            if (arrive) dc_red_release(bar_ctr, 1u);      // release: everything the bar.sync above ordered before it
            bar_target += n_arrivals;
            unsigned long long t0 = 0;
            int it = 0;
            while ((int)(dc_ld_acquire(bar_ctr) - bar_target) < 0) {
                if (((++it) & 0x3ff) == 0) {
                    const unsigned long long now = dc_timer();
                    if (!t0) t0 = now;
                    if (now - t0 > DC_TIMEOUT_NS || dc_ld_acquire(err_word)) {
                        atomicExch(err_word, 1u);
                        s_dead = 1;
                        break;
                    }
                }
            }
        }
        dc_bar(1, DC_CT);
        return s_dead == 0;
    };
    int seq = warp;     // this warp's next ring sequence number (advances by NW per stage, only for warp < NW)
    int gseq = 0;       // unit groups seen so far (index into the ticket ring s_gbase)
    // optional timeline: [2 CTAs][DC_MAX_JOBS + 1][4] stamps (job start, input staged, work done, dependency passed)
    const int tr_sel = blockIdx.x == 0 ? 0 : (blockIdx.x == gridDim.x - 1 ? 1 : -1);
    auto stamp = [&](int j, int k) {
        if (!p.trace || tid != 0) return;
        const unsigned long long now = dc_timer();
        if (tr_sel >= 0) p.trace[((size_t)tr_sel * (DC_MAX_JOBS + 1) + j) * 4 + k] = now;
        if (k == 2 && j < DC_MAX_JOBS) p.trace[2 * (DC_MAX_JOBS + 1) * 4 + (size_t)j * 160 + blockIdx.x] = now;   // every CTA: work done
    };
    stamp(DC_MAX_JOBS, 0);

    // activations come from the previous kernel: wait for it (no-op without the PDL attribute); the producer warp
    // above streams weights, which nobody writes, without waiting
    asm volatile("griddepcontrol.wait;" ::: "memory");
    stamp(DC_MAX_JOBS, 1);

    for (int j = 0; j < p.n_jobs; ++j) {
        const tl_decode_job& jb = p.jobs[j];
        const bool last_job = j == p.n_jobs - 1;
        stamp(j, 0);
        if (jb.type == TL_JOB_GEMV) {
            const int N = jb.N, K = jb.K, flags = jb.flags;
            const bf16* x = reinterpret_cast<const bf16*>(jb.x);
            bf16* y = reinterpret_cast<bf16*>(jb.y);
            const bf16* bias = reinterpret_cast<const bf16*>(jb.bias);
            const bf16* residual = reinterpret_cast<const bf16*>(jb.residual);
            const bf16* norm_w = reinterpret_cast<const bf16*>(jb.norm_w);
            const float eps = jb.eps;
            const int nvec = K >> 3;
            // ---- stage x (possibly written by other CTAs in the previous job: L2-coherent loads), one global pass
            // (the L2-coherent loads are volatile asm: issued in batches of 4 before anything consumes them, otherwise
            //  every iteration would pay a full L2 round trip in sequence)
            if (norm_w) {
                float ss[M];
#pragma unroll
                for (int m = 0; m < M; ++m) ss[m] = 0.f;
                constexpr int TB = M == 1 ? 4 : (M == 2 ? 2 : 1);
                for (int v0 = tid; v0 < nvec; v0 += TB * DC_CT) {
                    uint4 u[M][TB];
#pragma unroll
                    for (int m = 0; m < M; ++m)
#pragma unroll
                        for (int t = 0; t < TB; ++t)
                            if (v0 + t * DC_CT < nvec) u[m][t] = dc_ldcg_v4(x + (size_t)m * K + (size_t)(v0 + t * DC_CT) * 8);
#pragma unroll
                    for (int m = 0; m < M; ++m)
#pragma unroll
                        for (int t = 0; t < TB; ++t) {
                            const int v = v0 + t * DC_CT;
                            if (v < nvec) {
                                reinterpret_cast<uint4*>(xs + (size_t)m * K)[v] = u[m][t];
                                const uint32_t* u32 = reinterpret_cast<const uint32_t*>(&u[m][t]);
#pragma unroll
                                for (int q = 0; q < 4; ++q) {
                                    const float a = bf16_lo(u32[q]), b = bf16_hi(u32[q]);
                                    ss[m] += a * a + b * b;
                                }
                            }
                        }
                }
#pragma unroll
                for (int m = 0; m < M; ++m) {
                    const float t = warp_sum(ss[m]);
                    if (lane == 0) s_part[warp][m] = t;
                }
                dc_bar(1, DC_CT);
                float rstd[M];
#pragma unroll
                for (int m = 0; m < M; ++m) {
                    float t = 0.f;
#pragma unroll
                    for (int w = 0; w < DC_CW; ++w) t += s_part[w][m];
                    rstd[m] = 1.0f / sqrtf(t / (float)K + eps);
                }
                for (int v = tid; v < nvec; v += DC_CT) {          // each thread re-reads exactly what it wrote
                    const uint4 g = reinterpret_cast<const uint4*>(norm_w)[v];
                    const uint32_t* g32 = reinterpret_cast<const uint32_t*>(&g);
#pragma unroll
                    for (int m = 0; m < M; ++m) {
                        const uint4 u = reinterpret_cast<const uint4*>(xs + (size_t)m * K)[v];
                        uint4 o;
                        const uint32_t* u32 = reinterpret_cast<const uint32_t*>(&u);
                        uint32_t* o32 = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
                        for (int q = 0; q < 4; ++q)
                            o32[q] = pack_bf16(bf16_lo(g32[q]) * rbf(bf16_lo(u32[q]) * rstd[m]),
                                               bf16_hi(g32[q]) * rbf(bf16_hi(u32[q]) * rstd[m]));
                        reinterpret_cast<uint4*>(xs + (size_t)m * K)[v] = o;
                    }
                }
            } else {
                const int tot = nvec * M;
                for (int v0 = tid; v0 < tot; v0 += 4 * DC_CT) {
                    uint4 u[4];
#pragma unroll
                    for (int t = 0; t < 4; ++t)
                        if (v0 + t * DC_CT < tot) u[t] = dc_ldcg_v4(x + (size_t)(v0 + t * DC_CT) * 8);
#pragma unroll
                    for (int t = 0; t < 4; ++t)
                        if (v0 + t * DC_CT < tot) reinterpret_cast<uint4*>(xs)[v0 + t * DC_CT] = u[t];
                }
            }
            dc_bar(1, DC_CT);
            stamp(j, 1);

            const DcGeom g = dc_geom(N, K, DC_STAGE, DC_KC);
            const int u_end = p.dynamic ? g.U : g.u_end;
            const bool swiglu = flags & TL_EPI_SWIGLU;
            const int n_out = swiglu ? g.npairs : N;
            // bias / residual of a pair are fetched by lane 0 BEFORE the dot product (their L2 round trip would otherwise
            // sit between the last FMA and the store of every unit)
            auto preload = [&](int pair, float (&bs)[2], float (&rs)[M][2]) {
                bs[0] = bs[1] = 0.f;
#pragma unroll
                for (int m = 0; m < M; ++m) rs[m][0] = rs[m][1] = 0.f;
                if (lane != 0) return;
                const int r0 = 2 * pair;
                if (flags & TL_EPI_BIAS) {
                    bs[0] = bf2f(bias[r0]);
                    bs[1] = bf2f(bias[r0 + 1]);
                }
                if (flags & TL_EPI_RESIDUAL) {
#pragma unroll
                    for (int m = 0; m < M; ++m) {
                        rs[m][0] = dc_ldcg_bf16(residual + (size_t)m * N + r0);
                        rs[m][1] = dc_ldcg_bf16(residual + (size_t)m * N + r0 + 1);
                    }
                }
            };
            auto finish = [&](int pair, const float (&a0)[M], const float (&a1)[M], const float (&bs)[2], const float (&rs)[M][2]) {
                if (lane != 0) return;
                const int r0 = 2 * pair;
#pragma unroll
                for (int m = 0; m < M; ++m) {
                    float v0 = a0[m], v1 = a1[m];
                    if (flags & TL_EPI_BIAS) {
                        v0 += bs[0];
                        v1 += bs[1];
                    }
                    if (swiglu) {
                        const float gate = rbf(v0), up = rbf(v1);
                        y[(size_t)m * n_out + pair] = f2bf(rbf(silu_f(gate)) * up);
                    } else {
                        float t0 = rbf(v0), t1 = rbf(v1);
                        if (flags & TL_EPI_RESIDUAL) {
                            t0 += rs[m][0];
                            t1 += rs[m][1];
                        }
                        *reinterpret_cast<uint32_t*>(y + (size_t)m * N + r0) = pack_bf16(t0, t1);
                    }
                }
            };
            auto dot2 = [&](const uint4* r0, const uint4* r1, int k0, int vecs, float (&a0)[M], float (&a1)[M]) {
#pragma unroll 4
                for (int v = lane; v < vecs; v += 32) {
                    const uint4 w0 = r0[v], w1 = r1[v];
                    const uint32_t* a32 = reinterpret_cast<const uint32_t*>(&w0);
                    const uint32_t* b32 = reinterpret_cast<const uint32_t*>(&w1);
#pragma unroll
                    for (int m = 0; m < M; ++m) {
                        const uint4 xv = reinterpret_cast<const uint4*>(xs + (size_t)m * K + k0)[v];
                        const uint32_t* x32 = reinterpret_cast<const uint32_t*>(&xv);
#pragma unroll
                        for (int q = 0; q < 4; ++q) {
                            const float xl = bf16_lo(x32[q]), xh = bf16_hi(x32[q]);
                            a0[m] = fmaf(bf16_lo(a32[q]), xl, a0[m]);
                            a0[m] = fmaf(bf16_hi(a32[q]), xh, a0[m]);
                            a1[m] = fmaf(bf16_lo(b32[q]), xl, a1[m]);
                            a1[m] = fmaf(bf16_hi(b32[q]), xh, a1[m]);
                        }
                    }
                }
            };
            long long cwait = 0;
            const long long cjob0 = clock64();
            if (warp < NW) {
                for (;;) {                                   // unit groups until the producer's terminator group
                    int stage = seq % n_stages;
                    uint32_t phase = (uint32_t)(seq / n_stages) & 1u;
                    long long tw0 = clock64();
                    mbar_wait(&full_bar[stage], phase);
                    cwait += clock64() - tw0;
                    const int base = s_gbase[gseq & (DC_GB - 1)];
                    ++gseq;
                    if (base < 0) {                          // terminator: one empty stage per warp
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&empty_bar[stage]);
                        seq += NW;
                        break;
                    }
                    const int unit = base + warp;
                    const bool valid = unit < u_end;
                    const int pair0 = unit * g.P;
                    float a0[M], a1[M];
                    float bs[2], rs[M][2];
#pragma unroll
                    for (int m = 0; m < M; ++m) a0[m] = a1[m] = 0.f;
                    if (valid) preload(pair0, bs, rs);
                    for (int c = 0; c < g.n_chunks; ++c, seq += NW) {
                        if (c) {
                            stage = seq % n_stages;
                            phase = (uint32_t)(seq / n_stages) & 1u;
                            tw0 = clock64();
                            mbar_wait(&full_bar[stage], phase);
                            cwait += clock64() - tw0;
                        }
                        const unsigned char* src = ring + (size_t)stage * DC_STAGE;
                        if (valid) {
                            if (!g.chunked) {
                                const int np = min(g.P, g.npairs - pair0);
                                for (int pp = 0; pp < np; ++pp) {
                                    float b0[M], b1[M];
                                    float bn[2], rn[M][2];
#pragma unroll
                                    for (int m = 0; m < M; ++m) b0[m] = b1[m] = 0.f;
                                    if (pp + 1 < np) preload(pair0 + pp + 1, bn, rn);   // next pair's, under this pair's FMAs
                                    dot2(reinterpret_cast<const uint4*>(src + (size_t)(2 * pp) * K * 2),
                                         reinterpret_cast<const uint4*>(src + (size_t)(2 * pp + 1) * K * 2), 0, nvec, b0, b1);
#pragma unroll
                                    for (int m = 0; m < M; ++m) { b0[m] = warp_sum(b0[m]); b1[m] = warp_sum(b1[m]); }
                                    finish(pair0 + pp, b0, b1, bs, rs);
                                    if (pp + 1 < np) {
                                        bs[0] = bn[0]; bs[1] = bn[1];
#pragma unroll
                                        for (int m = 0; m < M; ++m) { rs[m][0] = rn[m][0]; rs[m][1] = rn[m][1]; }
                                    }
                                }
                            } else {
                                const int k0 = c * g.KC;
                                dot2(reinterpret_cast<const uint4*>(src), reinterpret_cast<const uint4*>(src + (size_t)g.KC * 2), k0,
                                     min(g.KC, K - k0) >> 3, a0, a1);
                            }
                        }
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&empty_bar[stage]);
                    }
                    if (valid && g.chunked) {
#pragma unroll
                        for (int m = 0; m < M; ++m) { a0[m] = warp_sum(a0[m]); a1[m] = warp_sum(a1[m]); }
                        finish(pair0, a0, a1, bs, rs);
                    }
                }
            }
            if (p.trace && blockIdx.x == 0 && tid == 0) {       // warp 0: cycles waiting for weights vs total cycles in the job's loop
                p.trace[DC_STAT_OFF + (size_t)j * 4 + 0] = (unsigned long long)cwait;
                p.trace[DC_STAT_OFF + (size_t)j * 4 + 1] = (unsigned long long)(clock64() - cjob0);
            }
            stamp(j, 2);
            if (!last_job && !grid_dep(true, gridDim.x)) break;
            stamp(j, 3);
        } else if (jb.type == TL_JOB_ATTN) {
            // ---- RoPE (+ q/k norm) + KV append + split-KV attention over all CTAs, one (row, kv head) group at a time.
            // Inside a CTA warp r owns query head r of the group end to end (scores with lane = key, online softmax in
            // registers, P.V with lane = output dims), so the only CTA-wide synchronisation is around the K/V tile in
            // shared memory; the tile's global loads are issued before anything else and fly under the q round trip.
            const int n_h = jb.n_h, n_kv = jb.n_kv, D = jb.d, T_max = jb.T_max;
            const int HALF = D >> 1, n_rep = n_h / n_kv;
            const int G = n_kv * M;
            const int cpg = (int)gridDim.x / G;                       // CTAs per group (>= 1, checked on the host)
            const int grp = (int)blockIdx.x / cpg, split = (int)blockIdx.x % cpg;
            const bool in_grid = grp < G;
            const int b = in_grid ? grp / n_kv : 0, kvh = in_grid ? grp % n_kv : 0;
            const int pos = reinterpret_cast<const int32_t*>(jb.pos_dev)[(jb.flags & TL_ATTN_POS_PER_ROW) ? b : 0];
            const int n_keys = pos + 1;                               // cached keys 0..pos-1 + the new token
            int cpg_eff = min(cpg, (n_keys + DC_MIN_KEYS - 1) / DC_MIN_KEYS);
            const int chunk = (((n_keys + cpg_eff - 1) / cpg_eff) + DC_TILE - 1) / DC_TILE * DC_TILE;   // whole tiles
            cpg_eff = (n_keys + chunk - 1) / chunk;                   // no empty ranges
            const bool active = in_grid && split < cpg_eff;
            float* sq = reinterpret_cast<float*>(attn_s);             // [8][128]
            float* sk = sq + 8 * 128;                                 // [128]
            float* sv = sk + 128;                                     // [128]
            float* sp = sv + 128;                                     // [8][DC_TILE]
            unsigned char* kt = reinterpret_cast<unsigned char*>(sp + 8 * DC_TILE);   // [DC_TILE][KT] bf16 rows, padded
            unsigned char* vt = kt + DC_TILE * DC_KT_MAX;
            const int KT = D * 2 + 16;                                // bytes per tile row
            if (tid == 0) s_last = 0;
            if (active) {
                const int k0 = split * chunk, k1 = min(n_keys, k0 + chunk);
                const bool owns_pos = k1 == n_keys;
                const int n_tiles = (k1 - k0 + DC_TILE - 1) / DC_TILE;
                const int heads = n_h + 2 * n_kv;
                const bf16* row = reinterpret_cast<const bf16*>(jb.x) + (size_t)b * heads * D;
                const bf16* cos_tab = reinterpret_cast<const bf16*>(jb.cos_tab);
                const bf16* sin_tab = reinterpret_cast<const bf16*>(jb.sin_tab);
                const bf16* qn = reinterpret_cast<const bf16*>(jb.q_norm_w);
                const bf16* kn = reinterpret_cast<const bf16*>(jb.k_norm_w);
                bf16* k_cache = reinterpret_cast<bf16*>(jb.k_cache);
                bf16* v_cache = reinterpret_cast<bf16*>(jb.v_cache);
                const bf16* kb = k_cache + ((size_t)b * n_kv + kvh) * T_max * D;
                const bf16* vb = v_cache + ((size_t)b * n_kv + kvh) * T_max * D;
                // tile loader: thread -> (row, 8-element column) of the [32, D] tile; 2 rows per thread at d = 128
                const int vpr = D >> 3, rpp = DC_CT / vpr, n_pass = DC_TILE / rpp;     // 16/16/2 or 8/32/1
                const int l_row = tid / vpr, l_col = (tid % vpr) * 8;
                uint4 kreg[2], vreg[2];
                auto load_tile = [&](int t0) {           // keys t0 .. t0+31 of the cache (rows >= pos are not in the cache)
#pragma unroll
                    for (int ps = 0; ps < 2; ++ps) {
                        kreg[ps] = make_uint4(0u, 0u, 0u, 0u);
                        vreg[ps] = make_uint4(0u, 0u, 0u, 0u);
                        const int key = t0 + ps * rpp + l_row;
                        if (ps < n_pass && key < k1 && key < pos) {
                            kreg[ps] = *reinterpret_cast<const uint4*>(kb + (size_t)key * D + l_col);
                            vreg[ps] = *reinterpret_cast<const uint4*>(vb + (size_t)key * D + l_col);
                        }
                    }
                };
                load_tile(k0);                           // in flight while q / k are fetched and rotated
                // -- q of the n_rep heads (warp u), k of the new token (warp n_rep) -> norm -> RoPE -> shared memory
                for (int u = warp; u <= n_rep; u += DC_CW) {
                    const bool is_k = u == n_rep;
                    if (is_k && !owns_pos) continue;
                    const bf16* src = row + (size_t)(is_k ? n_h + kvh : kvh * n_rep + u) * D;
                    const bf16* nw = is_k ? kn : qn;
                    float* dst = is_k ? sk : sq + u * 128;
                    float x1[2], x2[2], cs[2], sn[2];
                    float ssq = 0.f;
#pragma unroll
                    for (int t = 0; t < 2; ++t) {
                        const int i = lane + 32 * t;
                        x1[t] = x2[t] = cs[t] = sn[t] = 0.f;
                        if (i < HALF) {
                            x1[t] = dc_ldcg_bf16(src + i);
                            x2[t] = dc_ldcg_bf16(src + i + HALF);
                            cs[t] = bf2f(cos_tab[(size_t)pos * HALF + i]);
                            sn[t] = bf2f(sin_tab[(size_t)pos * HALF + i]);
                        }
                    }
#pragma unroll
                    for (int t = 0; t < 2; ++t) ssq += x1[t] * x1[t] + x2[t] * x2[t];
                    if (nw) {
                        const float r = 1.0f / sqrtf(warp_sum(ssq) / (float)D + jb.eps);
#pragma unroll
                        for (int t = 0; t < 2; ++t) {
                            const int i = lane + 32 * t;
                            if (i < HALF) {
                                x1[t] = rbf(bf2f(nw[i]) * rbf(x1[t] * r));
                                x2[t] = rbf(bf2f(nw[i + HALF]) * rbf(x2[t] * r));
                            }
                        }
                    }
#pragma unroll
                    for (int t = 0; t < 2; ++t) {
                        const int i = lane + 32 * t;
                        if (i < HALF) {
                            dst[i] = rbf(rbf(x1[t] * cs[t]) + rbf(-x2[t] * sn[t]));
                            dst[i + HALF] = rbf(rbf(x2[t] * cs[t]) + rbf(x1[t] * sn[t]));
                        }
                    }
                }
                if (owns_pos && tid < D) sv[tid] = dc_ldcg_bf16(row + (size_t)(n_h + n_kv + kvh) * D + tid);
                dc_bar(1, DC_CT);
                if (owns_pos && tid < D) {                       // append the new key / value to the cache
                    const size_t off = (((size_t)b * n_kv + kvh) * T_max + pos) * D + tid;
                    k_cache[off] = f2bf(sk[tid]);
                    v_cache[off] = f2bf(sv[tid]);
                }
                const float scale_log2 = jb.scale * 1.4426950408889634f;
                float m_run = -INFINITY, l_run = 0.f;
                float o[4] = {0.f, 0.f, 0.f, 0.f};
                for (int t = 0; t < n_tiles; ++t) {
                    const int t0 = k0 + t * DC_TILE;
                    // -- stage the tile (rows of the new token come from sk / sv, rows past the range stay zero)
#pragma unroll
                    for (int ps = 0; ps < 2; ++ps) {
                        if (ps < n_pass) {
                            const int r_ = ps * rpp + l_row, key = t0 + r_;
                            if (key == pos && key < k1) {
                                uint4 kk, vv;
                                uint32_t* k32 = reinterpret_cast<uint32_t*>(&kk);
                                uint32_t* v32 = reinterpret_cast<uint32_t*>(&vv);
#pragma unroll
                                for (int q = 0; q < 4; ++q) {
                                    k32[q] = pack_bf16(sk[l_col + 2 * q], sk[l_col + 2 * q + 1]);
                                    v32[q] = pack_bf16(sv[l_col + 2 * q], sv[l_col + 2 * q + 1]);
                                }
                                kreg[ps] = kk;
                                vreg[ps] = vv;
                            }
                            *reinterpret_cast<uint4*>(kt + (size_t)r_ * KT + l_col * 2) = kreg[ps];
                            *reinterpret_cast<uint4*>(vt + (size_t)r_ * KT + l_col * 2) = vreg[ps];
                        }
                    }
                    if (t + 1 < n_tiles) load_tile(t0 + DC_TILE);     // next tile's loads fly under this tile's math
                    dc_bar(1, DC_CT);
                    if (warp < n_rep) {
                        const int r = warp;
                        // scores: lane = key of the tile
                        float acc = 0.f;
                        const unsigned char* krow = kt + (size_t)lane * KT;
                        for (int c = 0; c < (D >> 3); ++c) {
                            const uint4 kv4 = *reinterpret_cast<const uint4*>(krow + c * 16);
                            const uint32_t* k32 = reinterpret_cast<const uint32_t*>(&kv4);
                            const float4 qa = *reinterpret_cast<const float4*>(&sq[r * 128 + c * 8]);
                            const float4 qb = *reinterpret_cast<const float4*>(&sq[r * 128 + c * 8 + 4]);
                            acc += bf16_lo(k32[0]) * qa.x + bf16_hi(k32[0]) * qa.y + bf16_lo(k32[1]) * qa.z + bf16_hi(k32[1]) * qa.w +
                                   bf16_lo(k32[2]) * qb.x + bf16_hi(k32[2]) * qb.y + bf16_lo(k32[3]) * qb.z + bf16_hi(k32[3]) * qb.w;
                        }
                        const bool in_range = t0 + lane < k1;
                        const float sc_ = in_range ? acc * scale_log2 : -INFINITY;
                        const float m_new = fmaxf(m_run, warp_max(sc_));          // finite: a tile always holds >= 1 key
                        const float pr = in_range ? exp2f(sc_ - m_new) : 0.f;
                        const float alpha = exp2f(m_run - m_new);                 // 0 on the first tile (m_run = -inf)
                        l_run = l_run * alpha + warp_sum(pr);
                        m_run = m_new;
                        sp[r * DC_TILE + lane] = rbf(pr);       // P is cast to bf16 before P.V (SDPA contract); l keeps fp32
                        __syncwarp();
                        // P.V: lane = D/32 output dims
#pragma unroll
                        for (int q = 0; q < 4; ++q) o[q] *= alpha;
                        if (D == 128) {
#pragma unroll 8
                            for (int key = 0; key < DC_TILE; ++key) {
                                const uint2 vv = *reinterpret_cast<const uint2*>(vt + (size_t)key * KT + lane * 8);
                                const float pk = sp[r * DC_TILE + key];
                                o[0] = fmaf(pk, bf16_lo(vv.x), o[0]);
                                o[1] = fmaf(pk, bf16_hi(vv.x), o[1]);
                                o[2] = fmaf(pk, bf16_lo(vv.y), o[2]);
                                o[3] = fmaf(pk, bf16_hi(vv.y), o[3]);
                            }
                        } else {
#pragma unroll 8
                            for (int key = 0; key < DC_TILE; ++key) {
                                const uint32_t vv = *reinterpret_cast<const uint32_t*>(vt + (size_t)key * KT + lane * 4);
                                const float pk = sp[r * DC_TILE + key];
                                o[0] = fmaf(pk, bf16_lo(vv), o[0]);
                                o[1] = fmaf(pk, bf16_hi(vv), o[1]);
                            }
                        }
                        __syncwarp();
                    }
                    if (t + 1 < n_tiles) dc_bar(1, DC_CT);          // the next staging overwrites the tile
                }
                const int EPL = D >> 5;                              // output dims per lane (4 or 2)
                if (cpg_eff == 1) {
                    // the only CTA of its group: the attention output of its heads goes out directly
                    if (warp < n_rep) {
                        bf16* yo = reinterpret_cast<bf16*>(jb.y) + ((size_t)b * n_h + kvh * n_rep + warp) * D + lane * EPL;
                        const float inv = 1.0f / l_run;
                        *reinterpret_cast<uint32_t*>(yo) = pack_bf16(o[0] * inv, o[1] * inv);
                        if (D == 128) *reinterpret_cast<uint32_t*>(yo + 2) = pack_bf16(o[2] * inv, o[3] * inv);
                    }
                    if (tid == 0) s_last = 1;
                } else {
                    // publish this CTA's partial (o unnormalised, m, l) per query head
                    if (warp < n_rep) {
                        float* pp = p.attn_part + (((size_t)b * n_h + kvh * n_rep + warp) * cpg + split) * (D + 4);
                        if (D == 128) *reinterpret_cast<float4*>(pp + lane * 4) = make_float4(o[0], o[1], o[2], o[3]);
                        else *reinterpret_cast<float2*>(pp + lane * 2) = make_float2(o[0], o[1]);
                        if (lane == 0) { pp[D] = m_run; pp[D + 1] = l_run; }
                    }
                    dc_bar(1, DC_CT);
                    if (tid == 0) {
                        __threadfence();
                        const unsigned old = atomicAdd(&grp_ctr[grp], 1u);
                        if (old == (unsigned)(cpg_eff - 1)) {
                            __threadfence();
                            s_last = 1;
                        }
                    }
                    dc_bar(1, DC_CT);
                    if (s_last) {
                        // the last CTA of the group combines the partials of all key ranges (batches of 4 independent loads)
                        if (warp < n_rep) {
                            const int h = kvh * n_rep + warp;
                            const float* base = p.attn_part + ((size_t)b * n_h + h) * cpg * (D + 4);
                            float mc = -INFINITY, L = 0.f, O[4] = {0.f, 0.f, 0.f, 0.f};
                            for (int s0 = 0; s0 < cpg_eff; s0 += 4) {
                                float ms[4], ls[4], os[4][4];
#pragma unroll
                                for (int q = 0; q < 4; ++q) {
                                    const int s_ = min(s0 + q, cpg_eff - 1);
                                    const float* e = base + (size_t)s_ * (D + 4);
                                    ms[q] = __ldcg(e + D);
                                    ls[q] = __ldcg(e + D + 1);
                                    if (D == 128) {
                                        const float4 t4 = __ldcg(reinterpret_cast<const float4*>(e + lane * 4));
                                        os[q][0] = t4.x; os[q][1] = t4.y; os[q][2] = t4.z; os[q][3] = t4.w;
                                    } else {
                                        const float2 t2 = __ldcg(reinterpret_cast<const float2*>(e + lane * 2));
                                        os[q][0] = t2.x; os[q][1] = t2.y; os[q][2] = os[q][3] = 0.f;
                                    }
                                }
#pragma unroll
                                for (int q = 0; q < 4; ++q) {
                                    if (s0 + q < cpg_eff) {
                                        const float mn = fmaxf(mc, ms[q]);
                                        const float a = exp2f(mc - mn), w = exp2f(ms[q] - mn);
                                        L = L * a + w * ls[q];
#pragma unroll
                                        for (int e_ = 0; e_ < 4; ++e_) O[e_] = O[e_] * a + w * os[q][e_];
                                        mc = mn;
                                    }
                                }
                            }
                            bf16* yo = reinterpret_cast<bf16*>(jb.y) + ((size_t)b * n_h + h) * D + lane * EPL;
                            const float inv = 1.0f / L;
                            *reinterpret_cast<uint32_t*>(yo) = pack_bf16(O[0] * inv, O[1] * inv);
                            if (D == 128) *reinterpret_cast<uint32_t*>(yo + 2) = pack_bf16(O[2] * inv, O[3] * inv);
                        }
                        if (tid == 0) grp_ctr[grp] = 0u;
                    }
                }
            }
            // one arrival per (row, kv head) group, by the CTA that wrote its output; everybody waits for all groups
            stamp(j, 2);
            if (!last_job && !grid_dep(s_last != 0, (unsigned)G)) break;
            stamp(j, 3);
        }
    }
    // ---- self-cleaning: the last CTA to leave resets the counters for the next launch on this sync slot
    dc_bar(1, DC_CT);
    stamp(DC_MAX_JOBS, 2);
    // (a producer parked on an empty-slot wait polls s_dead and leaves by itself)
    if (tid == 0 && last_cta_out(&p.sync[1])) {
        p.sync[0] = 0;
        for (int j = 0; j < p.n_jobs; ++j) p.sync[DC_JOBCTR + j] = 0;
        __threadfence();
    }
}

}  // namespace tl

static unsigned long long* g_chain_trace = nullptr;
static int g_chain_trace_slots = 0, g_chain_trace_next = 0;
constexpr int DC_TRACE_WORDS = tl::DC_STAT_OFF + tl::DC_MAX_JOBS * 4;

extern "C" {

/* debugging aid (tools/trace_chain.py): device buffer of n_slots * 2*(16+1)*4 uint64; every later chain launch takes the
 * next slot (a captured graph keeps its slots) and stamps it with globaltimer values (CTA 0 and the last CTA, per job:
 * start / input staged / work done / dependency passed; row 16: kernel entry / previous grid done / exit); NULL = off */
int tl_decode_chain_trace(void* buf, int n_slots) {
    g_chain_trace = (unsigned long long*)buf;
    g_chain_trace_slots = buf ? n_slots : 0;
    g_chain_trace_next = 0;
    return TL_OK;
}

size_t tl_decode_chain_ws(int M, int n_h, int n_kv, int d) {
    // attention partials [M*n_h][cpg][d+4] floats with cpg = CTAs / (n_kv*M) <= 160 / (n_kv*M) (160 bounds the SM count of every supported part)
    if (M < 1 || n_h < 1 || n_kv < 1) return 0;
    const int cpg = 160 / (n_kv * M) > 0 ? 160 / (n_kv * M) : 1;
    return (size_t)M * n_h * cpg * (d + 4) * sizeof(float) + 256;
}

static int chain_stage_kb() {       // TL_CHAIN_STAGE_KB, read once (any value below 8 but 0 forces 16 KB slots)
    static int forced_kb = -1;
    if (forced_kb < 0) {
        const char* e = getenv("TL_CHAIN_STAGE_KB");
        forced_kb = e ? atoi(e) : 0;
        if (forced_kb < 0) forced_kb = 16;
    }
    return forced_kb;
}

int tl_decode_chain_geometry(int M, int k_max, int stage_kb, int* out) {
    using namespace tl;
    TL_REQUIRE(M >= 1 && M <= DC_MAX_M && k_max >= 0 && out, TL_ERR_INVALID, "tl_decode_chain_geometry: M=%d k_max=%d", M, k_max);
    const int forced_kb = stage_kb < 0 ? chain_stage_kb() : stage_kb;
    constexpr int SMEM_CAP = 227 * 1024 - 1024;       // static shared memory of the kernel stays below 1 KB
    const size_t xs_bytes = (((size_t)M * k_max * 2) + 127) & ~(size_t)127;
    const size_t fixed = xs_bytes + (size_t)DC_ATTN_BYTES + 2 * DC_MAX_STAGES * sizeof(uint64_t);
    // The consumers are the scarce resource (one warp per scheduler cannot hide its own latencies), so all 8 consumer
    // warps get a slot class of their own: 8 slots (n_stages % NW == 0: a slot is always drained by the same warp) as
    // large as shared memory allows, capped at 24 KB.  Below 12 KB per slot, or with a forced slot size, as many slots
    // as fit, NW = the largest divisor-compatible warp count.
    int DC_STAGE = 0, n_stages = 0, NW = 0;
    TL_REQUIRE(fixed + 4 * 8192 <= (size_t)SMEM_CAP, TL_ERR_INVALID, "tl_decode_chain: M*K_max too large (%zu B fixed)", fixed);
    if (!forced_kb) {
        int kb = (int)((SMEM_CAP - fixed) / 8 / 1024);
        if (kb > 24) kb = 24;
        if (kb >= 12) { DC_STAGE = kb * 1024; n_stages = 8; NW = 8; }
    }
    if (!DC_STAGE) {
        DC_STAGE = (forced_kb >= 8 ? forced_kb : 16) * 1024;
        int max_stages = (int)((SMEM_CAP - fixed) / DC_STAGE);
        if (max_stages > DC_MAX_STAGES) max_stages = DC_MAX_STAGES;
        TL_REQUIRE(max_stages >= 4, TL_ERR_INVALID, "tl_decode_chain: fewer than 4 ring slots fit");
        for (int nw = DC_CW; nw >= 4; --nw) {
            const int st_ = max_stages / nw * nw;
            if (st_ > n_stages) { n_stages = st_; NW = nw; }
        }
    }
    out[0] = DC_STAGE;
    out[1] = n_stages;
    out[2] = NW;
    out[3] = (DC_STAGE / 4) & ~7;
    return TL_OK;
}

int tl_decode_chain(const tl_decode_job* jobs, int n_jobs, int M, void* sync_slot, void* attn_ws, size_t attn_ws_bytes,
                    const void* pf_ptr, size_t pf_bytes, void* stream) {
    using namespace tl;
    TL_REQUIRE(M >= 1 && M <= DC_MAX_M, TL_ERR_INVALID, "tl_decode_chain: M=%d outside 1..%d", M, DC_MAX_M);
    TL_REQUIRE(jobs && n_jobs > 0 && n_jobs <= DC_MAX_JOBS && sync_slot, TL_ERR_INVALID, "tl_decode_chain: bad job list (n=%d, max %d)",
               n_jobs, DC_MAX_JOBS);
    const int grid = sm_count();
    int k_max = 0, n_attn = 0;
    for (int j = 0; j < n_jobs; ++j) {
        const tl_decode_job& jb = jobs[j];
        if (jb.type == TL_JOB_GEMV) {
            TL_REQUIRE(jb.K % 8 == 0 && jb.N % 2 == 0 && jb.N > 0 && (((uintptr_t)jb.W) & 15) == 0, TL_ERR_INVALID,
                       "tl_decode_chain: job %d bad GEMV shape / alignment", j);
            if (jb.K > k_max) k_max = jb.K;
        } else if (jb.type == TL_JOB_ATTN) {
            TL_REQUIRE((jb.d == 64 || jb.d == 128) && jb.n_kv > 0 && jb.n_h % jb.n_kv == 0 && jb.n_h / jb.n_kv <= 8, TL_ERR_INVALID,
                       "tl_decode_chain: job %d attention shape unsupported (d=%d n_h=%d n_kv=%d)", j, jb.d, jb.n_h, jb.n_kv);
            const int G = jb.n_kv * M;
            TL_REQUIRE(G <= grid && G <= 60, TL_ERR_INVALID, "tl_decode_chain: %d (row, kv head) groups do not fit", G);
            const int cpg = grid / G;
            TL_REQUIRE(attn_ws && attn_ws_bytes >= (size_t)M * jb.n_h * cpg * (jb.d + 4) * sizeof(float), TL_ERR_INVALID,
                       "tl_decode_chain: attention workspace too small");
            ++n_attn;
        } else {
            TL_REQUIRE(false, TL_ERR_INVALID, "tl_decode_chain: job %d has unsupported type %d", j, jb.type);
        }
    }
    (void)n_attn;
    constexpr int SMEM_CAP = 227 * 1024 - 1024;
    const size_t xs_bytes = (((size_t)M * k_max * 2) + 127) & ~(size_t)127;
    const size_t fixed = xs_bytes + (size_t)DC_ATTN_BYTES + 2 * DC_MAX_STAGES * sizeof(uint64_t);
    int geo[4];
    if (tl_decode_chain_geometry(M, k_max, -1, geo) != TL_OK) return TL_ERR_INVALID;
    const int DC_STAGE = geo[0], n_stages = geo[1], NW = geo[2], DC_KC = geo[3];
    ChainParams prm = {};
    prm.n_jobs = n_jobs;
    prm.n_stages = n_stages;
    prm.NW = NW;
    prm.xs_bytes = (int)xs_bytes;
    static int dyn = -1, l2_ahead = -1;
    if (dyn < 0) {
        const char* e = getenv("TL_CHAIN_DYNAMIC");      // 1: units handed out by ticket counters instead of the static split
        dyn = (e && e[0] == '1') ? 1 : 0;                // (a ticket covers NW units, coarse at the tail)
        const char* a = getenv("TL_CHAIN_L2_AHEAD_KB");  // L2 prefetch lead per CTA; off by default
        l2_ahead = a ? atoi(a) * 1024 : 0;               // (a prefetch followed closely by the load of the same lines is fetched twice)
        if (l2_ahead < 0) l2_ahead = 0;
    }
    prm.dynamic = dyn;
    prm.stage_bytes = DC_STAGE;
    prm.kc = DC_KC;
    prm.l2_ahead = l2_ahead;
    prm.sync = (unsigned*)sync_slot;
    prm.attn_part = (float*)attn_ws;
    prm.pf_ptr = (const unsigned char*)pf_ptr;
    prm.pf_bytes = (((uintptr_t)pf_ptr) & 15) ? 0ull : (unsigned long long)(pf_bytes & ~(size_t)15);
    prm.trace = (g_chain_trace && g_chain_trace_next < g_chain_trace_slots)
                    ? g_chain_trace + (size_t)(g_chain_trace_next++) * DC_TRACE_WORDS : nullptr;
    for (int j = 0; j < n_jobs; ++j) prm.jobs[j] = jobs[j];
    const size_t smem = (size_t)n_stages * DC_STAGE + fixed;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(DC_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = (cudaStream_t)stream;
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
#define TL_DC_LAUNCH(MM)                                                                                                   \
    {                                                                                                                      \
        static bool done = false;                                                                                          \
        if (!done) {                                                                                                       \
            if (cudaFuncSetAttribute(decode_chain_kernel<MM>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_CAP) != cudaSuccess) \
                return check_launch("tl_decode_chain (smem attr)");                                                      \
            done = true;                                                                                                   \
        }                                                                                                                  \
        cudaLaunchKernelEx(&cfg, decode_chain_kernel<MM>, prm);                                                            \
    }
    switch (M) {
        case 1: TL_DC_LAUNCH(1) break;
        case 2: TL_DC_LAUNCH(2) break;
        case 3: TL_DC_LAUNCH(3) break;
        default: TL_DC_LAUNCH(4) break;
    }
#undef TL_DC_LAUNCH
    return check_launch("tl_decode_chain");
}

}  // extern "C"
