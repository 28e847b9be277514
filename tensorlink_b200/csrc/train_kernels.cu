// Training-only HBM-bound kernels (K8/K9/K10 of SURVEY.md §2.4): SwiGLU fwd/bwd on interleaved gate/up
// pre-activations, RMSNorm backward, RoPE(+KV scatter) backward, shifted cross-entropy forward+backward,
// embedding backward, bias column sums, gradient accumulation and a fused AdamW step.
// They replace the autograd graph of unfused ATen ops the reference's worker runs in
// `assoc_output.backward(loss)` (/root/reference/tensorlink/ml/worker.py:271) and its `optimizer.step()` (:1317).
#include <stdlib.h>

#include "common.cuh"

namespace tl {

// ------------------------------------------------------------------------------------------------ SwiGLU
// gu[M, 2I] interleaved (2j = gate_j, 2j+1 = up_j)  ->  h[M, I] = bf16(bf16(silu(g)) * u)     (HF rounding)
__global__ void swiglu_fwd_kernel(const uint4* __restrict__ gu, uint2* __restrict__ h, size_t n_vec) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += (size_t)gridDim.x * blockDim.x) {
        const uint4 v = gu[i];          // 4 (gate, up) pairs
        const uint32_t* p = reinterpret_cast<const uint32_t*>(&v);
        float o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) o[j] = rbf(silu_f(bf16_lo(p[j]))) * bf16_hi(p[j]);
        h[i] = make_uint2(pack_bf16(o[0], o[1]), pack_bf16(o[2], o[3]));
    }
}

// dgu from dh:  d_gate = dh * u * silu'(g),  d_up = dh * silu(g);  silu'(g) = s + g*s*(1-s), s = sigmoid(g)
__global__ void swiglu_bwd_kernel(const uint4* __restrict__ gu, const uint2* __restrict__ dh, uint4* __restrict__ dgu,
                                  size_t n_vec) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += (size_t)gridDim.x * blockDim.x) {
        const uint4 v = gu[i];
        const uint2 d = dh[i];
        const uint32_t* p = reinterpret_cast<const uint32_t*>(&v);
        const float dd[4] = {bf16_lo(d.x), bf16_hi(d.x), bf16_lo(d.y), bf16_hi(d.y)};
        uint32_t o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float g = bf16_lo(p[j]), u = bf16_hi(p[j]);
            const float s = 1.0f / (1.0f + expf(-g));
            const float act = rbf(g * s);                          // the bf16 silu(g) the forward multiplied by
            const float dact = rbf(dd[j] * u);                     // grad wrt silu output (bf16 like autograd)
            o[j] = pack_bf16(dact * (s + g * s * (1.0f - s)), dd[j] * act);
        }
        dgu[i] = make_uint4(o[0], o[1], o[2], o[3]);
    }
}

// ------------------------------------------------------------------------------------------------ RMSNorm backward
// n = x*rstd, g = dy*w:  dx = rstd * (g - n * mean(g*n)) [+ dx_add];  dw[h] += sum_rows dy*n
// (dw: one partial row per CTA in dw_part, summed in CTA order by det_reduce_kernel)
constexpr int NB_THREADS = 128;
template <int NB_MAXV>
__global__ void __launch_bounds__(NB_THREADS) rmsnorm_bwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                                                                   const bf16* __restrict__ dy, const float* __restrict__ rstd,
                                                                   const bf16* __restrict__ dx_add, bf16* __restrict__ dx,
                                                                   float* __restrict__ dw_part, int rows, int H,
                                                                   int rows_per_block) {
    const int nvec = H >> 3;
    float dwl[NB_MAXV][8];
#pragma unroll
    for (int i = 0; i < NB_MAXV; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) dwl[i][j] = 0.f;
    __shared__ float red[NB_THREADS / 32];
    const int r0 = blockIdx.x * rows_per_block, r1 = min(rows, r0 + rows_per_block);
    uint4 wreg[NB_MAXV];
#pragma unroll
    for (int i = 0; i < NB_MAXV; ++i) {
        const int idx = threadIdx.x + i * NB_THREADS;
        wreg[i] = idx < nvec ? reinterpret_cast<const uint4*>(w)[idx] : make_uint4(0, 0, 0, 0);
    }
    // the loads of row r+1 are issued before the two block barriers of row r (the row loop is otherwise one dependent
    // chain per row)
    uint4 xn[NB_MAXV], dn[NB_MAXV], an[NB_MAXV];
    auto fetch = [&](int row) {
        const uint4* xr = reinterpret_cast<const uint4*>(x + (size_t)row * H);
        const uint4* dr = reinterpret_cast<const uint4*>(dy + (size_t)row * H);
        const uint4* ar = dx_add ? reinterpret_cast<const uint4*>(dx_add + (size_t)row * H) : nullptr;
#pragma unroll
        for (int i = 0; i < NB_MAXV; ++i) {
            const int idx = threadIdx.x + i * NB_THREADS;
            if (idx < nvec) {
                xn[i] = xr[idx];
                dn[i] = dr[idx];
                an[i] = ar ? ar[idx] : make_uint4(0, 0, 0, 0);
            }
        }
    };
    if (r0 < r1) fetch(r0);
    for (int row = r0; row < r1; ++row) {
        const float rs = rstd[row];
        float nv[NB_MAXV][8], gv[NB_MAXV][8];
        uint4 av[NB_MAXV];
        float dot = 0.f;
#pragma unroll
        for (int i = 0; i < NB_MAXV; ++i) {
            const int idx = threadIdx.x + i * NB_THREADS;
            if (idx < nvec) {
                const uint4 xv = xn[i], dv = dn[i], wv = wreg[i];
                av[i] = an[i];
                const uint32_t* x32 = reinterpret_cast<const uint32_t*>(&xv);
                const uint32_t* d32 = reinterpret_cast<const uint32_t*>(&dv);
                const uint32_t* w32 = reinterpret_cast<const uint32_t*>(&wv);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float n0 = bf16_lo(x32[j]) * rs, n1 = bf16_hi(x32[j]) * rs;
                    const float d0 = bf16_lo(d32[j]), d1 = bf16_hi(d32[j]);
                    nv[i][2 * j] = n0; nv[i][2 * j + 1] = n1;
                    gv[i][2 * j] = d0 * bf16_lo(w32[j]); gv[i][2 * j + 1] = d1 * bf16_hi(w32[j]);
                    dot += gv[i][2 * j] * n0 + gv[i][2 * j + 1] * n1;
                    dwl[i][2 * j] += d0 * rbf(n0); dwl[i][2 * j + 1] += d1 * rbf(n1);
                }
            }
        }
        if (row + 1 < r1) fetch(row + 1);
        dot = warp_sum(dot);
        __syncthreads();
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = dot;
        __syncthreads();
        float tot = 0.f;
#pragma unroll
        for (int i = 0; i < NB_THREADS / 32; ++i) tot += red[i];
        const float mean = tot / (float)H;
        uint4* outr = reinterpret_cast<uint4*>(dx + (size_t)row * H);
#pragma unroll
        for (int i = 0; i < NB_MAXV; ++i) {
            const int idx = threadIdx.x + i * NB_THREADS;
            if (idx < nvec) {
                float o[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) o[j] = rbf(rs * (gv[i][j] - nv[i][j] * mean));
                if (dx_add) {
                    const uint32_t* a32 = reinterpret_cast<const uint32_t*>(&av[i]);
#pragma unroll
                    for (int j = 0; j < 4; ++j) { o[2 * j] += bf16_lo(a32[j]); o[2 * j + 1] += bf16_hi(a32[j]); }
                }
                outr[idx] = make_uint4(pack_bf16(o[0], o[1]), pack_bf16(o[2], o[3]), pack_bf16(o[4], o[5]), pack_bf16(o[6], o[7]));
            }
        }
    }
    if (dw_part) {
        float* dst = dw_part + (size_t)blockIdx.x * H;
#pragma unroll
        for (int i = 0; i < NB_MAXV; ++i) {
            const int idx = threadIdx.x + i * NB_THREADS;
            if (idx < nvec) {
#pragma unroll
                for (int j = 0; j < 8; ++j) dst[idx * 8 + j] = dwl[i][j];
            }
        }
    }
}


// narrow rows (H <= 1024): one WARP per row, 4 rows in flight per CTA, no block barriers in the row loop
constexpr int NBW_MAXV = 4;
__global__ void __launch_bounds__(NB_THREADS) rmsnorm_bwd_warp_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                                                                        const bf16* __restrict__ dy, const float* __restrict__ rstd,
                                                                        const bf16* __restrict__ dx_add, bf16* __restrict__ dx,
                                                                        float* __restrict__ dw_part, int rows, int H) {
    const int nvec = H >> 3, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int gw = blockIdx.x * (NB_THREADS / 32) + warp, nw = gridDim.x * (NB_THREADS / 32);
    float dwl[NBW_MAXV][8];
    uint4 wreg[NBW_MAXV];
#pragma unroll
    for (int i = 0; i < NBW_MAXV; ++i) {
        const int idx = lane + 32 * i;
        wreg[i] = idx < nvec ? reinterpret_cast<const uint4*>(w)[idx] : make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int j = 0; j < 8; ++j) dwl[i][j] = 0.f;
    }
    for (int row = gw; row < rows; row += nw) {
        const uint4* xr = reinterpret_cast<const uint4*>(x + (size_t)row * H);
        const uint4* dr = reinterpret_cast<const uint4*>(dy + (size_t)row * H);
        const float rs = rstd[row];
        float nv[NBW_MAXV][8], gv[NBW_MAXV][8];
        float dot = 0.f;
#pragma unroll
        for (int i = 0; i < NBW_MAXV; ++i) {
            const int idx = lane + 32 * i;
            if (idx < nvec) {
                const uint4 xv = xr[idx], dv = dr[idx];
                const uint32_t* x32 = reinterpret_cast<const uint32_t*>(&xv);
                const uint32_t* d32 = reinterpret_cast<const uint32_t*>(&dv);
                const uint32_t* w32 = reinterpret_cast<const uint32_t*>(&wreg[i]);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float n0 = bf16_lo(x32[j]) * rs, n1 = bf16_hi(x32[j]) * rs;
                    const float d0 = bf16_lo(d32[j]), d1 = bf16_hi(d32[j]);
                    nv[i][2 * j] = n0; nv[i][2 * j + 1] = n1;
                    gv[i][2 * j] = d0 * bf16_lo(w32[j]); gv[i][2 * j + 1] = d1 * bf16_hi(w32[j]);
                    dot += gv[i][2 * j] * n0 + gv[i][2 * j + 1] * n1;
                    dwl[i][2 * j] += d0 * rbf(n0); dwl[i][2 * j + 1] += d1 * rbf(n1);
                }
            }
        }
        const float mean = warp_sum(dot) / (float)H;
        uint4* outr = reinterpret_cast<uint4*>(dx + (size_t)row * H);
#pragma unroll
        for (int i = 0; i < NBW_MAXV; ++i) {
            const int idx = lane + 32 * i;
            if (idx < nvec) {
                float o[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) o[j] = rbf(rs * (gv[i][j] - nv[i][j] * mean));
                if (dx_add) {
                    const uint4 av = reinterpret_cast<const uint4*>(dx_add + (size_t)row * H)[idx];
                    const uint32_t* a32 = reinterpret_cast<const uint32_t*>(&av);
#pragma unroll
                    for (int j = 0; j < 4; ++j) { o[2 * j] += bf16_lo(a32[j]); o[2 * j + 1] += bf16_hi(a32[j]); }
                }
                outr[idx] = make_uint4(pack_bf16(o[0], o[1]), pack_bf16(o[2], o[3]), pack_bf16(o[4], o[5]), pack_bf16(o[6], o[7]));
            }
        }
    }
    if (dw_part) {
        __shared__ float sdw[NB_THREADS / 32][NBW_MAXV * 32 * 8 + 1];
#pragma unroll
        for (int i = 0; i < NBW_MAXV; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) sdw[warp][(lane + 32 * i) * 8 + j] = dwl[i][j];
        __syncthreads();
        for (int c = threadIdx.x; c < H; c += NB_THREADS) {
            float t = 0.f;
#pragma unroll
            for (int wv = 0; wv < NB_THREADS / 32; ++wv) t += sdw[wv][c];
            dw_part[(size_t)blockIdx.x * H + c] = t;
        }
    }
}

// ------------------------------------------------------------------------------------------------ RoPE backward
// one warp per (token, head): inverse rotation of dq / dk, plain gather of dv -> dqkv[n, (n_h+2n_kv)*d]
template <int D>
__global__ void __launch_bounds__(128) rope_kv_bwd_kernel(const bf16* __restrict__ dq, const bf16* __restrict__ dk,
                                                           const bf16* __restrict__ dv, bf16* __restrict__ dqkv,
                                                           const bf16* __restrict__ cos_tab, const bf16* __restrict__ sin_tab,
                                                           int n_tokens, int S, int n_h, int n_kv, int T_max) {
    constexpr int HALF = D / 2, PAIRS = HALF / 32;
    const int heads = n_h + 2 * n_kv;
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (gw >= n_tokens * heads) return;
    const int n = gw / heads, h = gw - n * heads;
    const int b = n / S, pos = n - b * S;
    bf16* dst = dqkv + (size_t)n * heads * D + (size_t)h * D;
    const bool is_q = h < n_h, is_k = !is_q && h < n_h + n_kv;
    // dk / dv arrive as one partial per QUERY head ([B, n_h, T_max, d]); the n_rep partials of a kv head are summed here
    const int n_rep = n_h / n_kv;
    const int kvh = is_q ? 0 : (is_k ? h - n_h : h - n_h - n_kv);
    const bf16* src = is_q ? dq + (size_t)n * n_h * D + (size_t)h * D
                           : (is_k ? dk : dv) + (((size_t)b * n_h + (size_t)kvh * n_rep) * T_max + pos) * D;
#pragma unroll
    for (int p = 0; p < PAIRS; ++p) {
        const int i = lane + 32 * p;
        float d1 = bf2f(src[i]), d2 = bf2f(src[i + HALF]);
        if (!is_q) {
            for (int r = 1; r < n_rep; ++r) {
                d1 += bf2f(src[(size_t)r * T_max * D + i]);
                d2 += bf2f(src[(size_t)r * T_max * D + i + HALF]);
            }
        }
        if (!is_q && !is_k) {
            dst[i] = f2bf(d1);
            dst[i + HALF] = f2bf(d2);
        } else {
            const float c = bf2f(cos_tab[(size_t)pos * HALF + i]), s = bf2f(sin_tab[(size_t)pos * HALF + i]);
            dst[i] = f2bf(d1 * c + d2 * s);
            dst[i + HALF] = f2bf(d2 * c - d1 * s);
        }
    }
}


// ------------------------------------------------------------------------------------------------ q/k-norm backward
// Qwen3: q and k heads are RMS-normalised over the head dim before RoPE (modeling_qwen3.py:248-264).  One warp per
// (token, q-or-k head): recompute rstd from the saved pre-norm qkv, replace the gradient slice of dqkv in place by
// the gradient w.r.t. the pre-norm vector, accumulate the gain gradients in fp32: warps stride over the items, and each
// CTA writes one partial row [q gains | k gains] to part (summed in CTA order by det_reduce_kernel).
template <int D>
__global__ void __launch_bounds__(128) qk_norm_bwd_kernel(const bf16* __restrict__ qkv_pre, bf16* __restrict__ dqkv,
                                                           const bf16* __restrict__ qn, const bf16* __restrict__ kn,
                                                           float* __restrict__ part, float eps, int n_tokens, int n_h, int n_kv) {
    constexpr int PER = D / 32;
    const int heads = n_h + 2 * n_kv, nh_qk = n_h + n_kv;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float accq[PER], acck[PER];
#pragma unroll
    for (int p = 0; p < PER; ++p) accq[p] = acck[p] = 0.f;
    for (long long item = (long long)blockIdx.x * 4 + warp; item < (long long)n_tokens * nh_qk; item += (long long)gridDim.x * 4) {
    const int n = (int)(item / nh_qk), h = (int)(item - (long long)n * nh_qk);
    const bool is_q = h < n_h;
    const size_t off = (size_t)n * heads * D + (size_t)h * D;
    const bf16* w = is_q ? qn : kn;
    float x[PER], g[PER], dy[PER];
    float ss = 0.f;
#pragma unroll
    for (int p = 0; p < PER; ++p) {
        x[p] = bf2f(qkv_pre[off + lane + 32 * p]);
        ss += x[p] * x[p];
    }
    ss = warp_sum(ss);
    const float rstd = 1.0f / sqrtf(ss / (float)D + eps);
    float dot = 0.f;
#pragma unroll
    for (int p = 0; p < PER; ++p) {
        dy[p] = bf2f(dqkv[off + lane + 32 * p]);
        g[p] = dy[p] * bf2f(w[lane + 32 * p]);
        dot += g[p] * x[p] * rstd;
    }
    dot = warp_sum(dot) / (float)D;
#pragma unroll
    for (int p = 0; p < PER; ++p) {
        const float nrm = x[p] * rstd;
        dqkv[off + lane + 32 * p] = f2bf(rstd * (g[p] - nrm * dot));
        if (is_q) accq[p] += dy[p] * rbf(nrm);
        else acck[p] += dy[p] * rbf(nrm);
    }
    }
    __shared__ float sp[4][2 * D];
#pragma unroll
    for (int p = 0; p < PER; ++p) {
        sp[warp][lane + 32 * p] = accq[p];
        sp[warp][D + lane + 32 * p] = acck[p];
    }
    __syncthreads();
    for (int c = threadIdx.x; c < 2 * D; c += blockDim.x)
        part[(size_t)blockIdx.x * 2 * D + c] = sp[0][c] + sp[1][c] + sp[2][c] + sp[3][c];
}

// ------------------------------------------------------------------------------------------------ cross entropy
// one CTA per row: loss_part[row] = logsumexp(row) - row[label] (0 for ignored rows; summed in row order by
// det_reduce_kernel); dlogits = (softmax - onehot) * grad_scale (in place ok)
constexpr int CE_THREADS = 512;
__global__ void __launch_bounds__(CE_THREADS) ce_fwd_bwd_kernel(const bf16* __restrict__ logits, const int64_t* __restrict__ labels,
                                                                 float* __restrict__ loss_part, int32_t* __restrict__ n_valid,
                                                                 bf16* __restrict__ dlogits, float grad_scale, int V) {
    const int row = blockIdx.x;
    const long long label = labels[row];
    const bf16* lr = logits + (size_t)row * V;
    bf16* dr = dlogits + (size_t)row * V;
    const int nvec = V >> 3;
    __shared__ float red[CE_THREADS / 32];
    __shared__ float s_bcast;
    if (label < 0 || label >= V) {      // ignore_index (-100): zero gradient, no loss
        if (threadIdx.x == 0) loss_part[row] = 0.f;
        if (dlogits) for (int i = threadIdx.x; i < nvec; i += CE_THREADS) reinterpret_cast<uint4*>(dr)[i] = make_uint4(0, 0, 0, 0);
        return;
    }
    float mx = -INFINITY;
    for (int i = threadIdx.x; i < nvec; i += CE_THREADS) {
        const uint4 v = reinterpret_cast<const uint4*>(lr)[i];
        const uint32_t* p = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
        for (int j = 0; j < 4; ++j) mx = fmaxf(mx, fmaxf(bf16_lo(p[j]), bf16_hi(p[j])));
    }
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x == 0) {
        float m = red[0];
        for (int i = 1; i < CE_THREADS / 32; ++i) m = fmaxf(m, red[i]);
        s_bcast = m;
    }
    __syncthreads();
    mx = s_bcast;
    float se = 0.f;
    for (int i = threadIdx.x; i < nvec; i += CE_THREADS) {
        const uint4 v = reinterpret_cast<const uint4*>(lr)[i];
        const uint32_t* p = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
        for (int j = 0; j < 4; ++j) se += expf(bf16_lo(p[j]) - mx) + expf(bf16_hi(p[j]) - mx);
    }
    se = warp_sum(se);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = se;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int i = 0; i < CE_THREADS / 32; ++i) s += red[i];
        s_bcast = s;
        const float lse = mx + logf(s);
        loss_part[row] = lse - bf2f(lr[label]);
        if (n_valid) atomicAdd(n_valid, 1);
    }
    __syncthreads();
    if (!dlogits) return;
    const float inv = grad_scale / s_bcast;
    for (int i = threadIdx.x; i < nvec; i += CE_THREADS) {
        const uint4 v = reinterpret_cast<const uint4*>(lr)[i];
        const uint32_t* p = reinterpret_cast<const uint32_t*>(&v);
        float o[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            o[2 * j] = expf(bf16_lo(p[j]) - mx) * inv;
            o[2 * j + 1] = expf(bf16_hi(p[j]) - mx) * inv;
        }
        const int base = i * 8;
        if (label >= base && label < base + 8) o[label - base] -= grad_scale;
        reinterpret_cast<uint4*>(dr)[i] = make_uint4(pack_bf16(o[0], o[1]), pack_bf16(o[2], o[3]), pack_bf16(o[4], o[5]), pack_bf16(o[6], o[7]));
    }
}

// ------------------------------------------------------------------------------------------------ embedding backward
// dtable[ids[t]] += dout[t].  The warp of the FIRST token carrying an id adds the rows of every token with that id, in
// token order (bf16 rounding after each add), so no two warps touch one table row and the result is the same every run.
__global__ void embed_bwd_kernel(const int64_t* __restrict__ ids, const bf16* __restrict__ dout, bf16* __restrict__ dtable,
                                 int n_tokens, int H, int vocab) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= n_tokens) return;
    const long long id = ids[warp];
    if (id < 0 || id >= vocab) return;
    for (int j0 = 0; j0 < warp; j0 += 32) {
        const int j = j0 + lane;
        if (__any_sync(0xffffffffu, j < warp && ids[j] == id)) return;   // an earlier token owns this row
    }
    __nv_bfloat162* dst = reinterpret_cast<__nv_bfloat162*>(dtable + (size_t)id * H);
    for (int j0 = warp; j0 < n_tokens; j0 += 32) {
        const int j = j0 + lane;
        unsigned m = __ballot_sync(0xffffffffu, j < n_tokens && ids[j] == id);
        while (m) {
            const int t = j0 + __ffs(m) - 1;
            m &= m - 1;
            const __nv_bfloat162* src = reinterpret_cast<const __nv_bfloat162*>(dout + (size_t)t * H);
            for (int i = lane; i < (H >> 1); i += 32) dst[i] = __hadd2(dst[i], src[i]);
        }
    }
}

// ------------------------------------------------------------------------------------------------ column sum (bias grad)
// db_accum[c] += sum_m dy[m, c].  block = 32x8 threads: 64 columns x a 256-row slab; the slab's sums go to row
// blockIdx.y of part [slabs][N] (summed in slab order by det_reduce_kernel)
__global__ void colsum_kernel(const bf16* __restrict__ dy, float* __restrict__ part, int M, int N, int ld) {
    const int c2 = blockIdx.x * 32 + threadIdx.x;      // bf16x2 column index
    float a0 = 0.f, a1 = 0.f;
    const int m0 = blockIdx.y * 256, m1 = min(M, m0 + 256);
    if (2 * c2 < N) {
        for (int m = m0 + threadIdx.y; m < m1; m += 8) {
            const uint32_t u = *reinterpret_cast<const uint32_t*>(dy + (size_t)m * ld + 2 * c2);
            a0 += bf16_lo(u);
            a1 += bf16_hi(u);
        }
    }
    __shared__ float s0[8][33], s1[8][33];
    s0[threadIdx.y][threadIdx.x] = a0;
    s1[threadIdx.y][threadIdx.x] = a1;
    __syncthreads();
    if (threadIdx.y == 0 && 2 * c2 < N) {
#pragma unroll
        for (int j = 1; j < 8; ++j) { a0 += s0[j][threadIdx.x]; a1 += s1[j][threadIdx.x]; }
        part[(size_t)blockIdx.y * N + 2 * c2] = a0;
        part[(size_t)blockIdx.y * N + 2 * c2 + 1] = a1;
    }
}

// fp32 accumulator -> bf16 gradient (+=)
__global__ void f32_to_bf16_accum_kernel(const float* __restrict__ src, bf16* __restrict__ dst, size_t n, int accumulate) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        dst[i] = f2bf(src[i] + (accumulate ? bf2f(dst[i]) : 0.f));
}

__global__ void add_inplace_kernel(uint4* __restrict__ a, const uint4* __restrict__ b, size_t n_vec) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += (size_t)gridDim.x * blockDim.x) {
        uint4 x = a[i];
        const uint4 y = b[i];
        uint32_t* x32 = reinterpret_cast<uint32_t*>(&x);
        const uint32_t* y32 = reinterpret_cast<const uint32_t*>(&y);
#pragma unroll
        for (int j = 0; j < 4; ++j) x32[j] = pack_bf16(bf16_lo(x32[j]) + bf16_lo(y32[j]), bf16_hi(x32[j]) + bf16_hi(y32[j]));
        a[i] = x;
    }
}

// a[i] = (accumulate ? a[i] : 0) + scale * b[i]  over bf16 (fp32 math, one rounding): commits a pending gradient
// (produced during the forward pass) into the gradient arena with the upstream gradient's scale
__global__ void scale_add_bf16_kernel(uint4* __restrict__ a, const uint4* __restrict__ b, float scale, int accumulate, size_t n_vec) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += (size_t)gridDim.x * blockDim.x) {
        uint4 x = accumulate ? a[i] : make_uint4(0u, 0u, 0u, 0u);
        const uint4 y = b[i];
        uint32_t* x32 = reinterpret_cast<uint32_t*>(&x);
        const uint32_t* y32 = reinterpret_cast<const uint32_t*>(&y);
#pragma unroll
        for (int j = 0; j < 4; ++j)
            x32[j] = pack_bf16(fmaf(scale, bf16_lo(y32[j]), bf16_lo(x32[j])), fmaf(scale, bf16_hi(y32[j]), bf16_hi(x32[j])));
        a[i] = x;
    }
}

__global__ void scale_add_f32_kernel(float* __restrict__ a, const float* __restrict__ b, float scale, int accumulate, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        a[i] = fmaf(scale, b[i], accumulate ? a[i] : 0.f);
}

// ------------------------------------------------------------------------------------------------ AdamW
// torch.optim.Adam/AdamW update rule in fp32 on bf16 parameters, fp32 moments
__device__ __forceinline__ void adamw_one(float& pw, float gr, float& mi, float& vi, float lr, float b1, float b2, float eps,
                                          float wd, float bc1, float bc2_sqrt, int decoupled) {
    if (wd != 0.f) {
        if (decoupled) pw *= (1.0f - lr * wd);
        else gr += wd * pw;
    }
    mi = b1 * mi + (1.0f - b1) * gr;
    vi = b2 * vi + (1.0f - b2) * gr * gr;
    const float denom = sqrtf(vi) / bc2_sqrt + eps;
    pw = pw - (lr / bc1) * (mi / denom);
}

// 8 elements per thread and iteration: 16-byte accesses to p / g, 2 x 16 bytes to each moment (22 bytes of HBM
// traffic per parameter: this sweep is 1/6 of a Qwen2.5-7B step at batch 8 x 512, so it has to run at copy speed)
template <bool STREAM>
__global__ void adamw_kernel(bf16* __restrict__ p, const bf16* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                             size_t n, float lr, float b1, float b2, float eps, float wd, float bc1, float bc2_sqrt,
                             int decoupled) {
    const size_t n8 = n >> 3;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += stride) {
        uint4 pu, gu;
        float4 m0, m1, v0, v1;
        if (STREAM) {   // every byte is touched once per step: evict-first loads and stores keep L2 for nothing
            pu = __ldcs(reinterpret_cast<const uint4*>(p) + i);
            gu = __ldcs(reinterpret_cast<const uint4*>(g) + i);
            m0 = __ldcs(reinterpret_cast<const float4*>(m) + 2 * i); m1 = __ldcs(reinterpret_cast<const float4*>(m) + 2 * i + 1);
            v0 = __ldcs(reinterpret_cast<const float4*>(v) + 2 * i); v1 = __ldcs(reinterpret_cast<const float4*>(v) + 2 * i + 1);
        } else {
            pu = reinterpret_cast<const uint4*>(p)[i];
            gu = ldg_nc_v4(reinterpret_cast<const uint4*>(g) + i);
            m0 = reinterpret_cast<const float4*>(m)[2 * i]; m1 = reinterpret_cast<const float4*>(m)[2 * i + 1];
            v0 = reinterpret_cast<const float4*>(v)[2 * i]; v1 = reinterpret_cast<const float4*>(v)[2 * i + 1];
        }
        uint32_t* p32 = reinterpret_cast<uint32_t*>(&pu);
        const uint32_t* g32 = reinterpret_cast<const uint32_t*>(&gu);
        float* mm[2] = {reinterpret_cast<float*>(&m0), reinterpret_cast<float*>(&m1)};
        float* vv[2] = {reinterpret_cast<float*>(&v0), reinterpret_cast<float*>(&v1)};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float pa = bf16_lo(p32[j]), pb = bf16_hi(p32[j]);
            float* mj = mm[j >> 1] + 2 * (j & 1);
            float* vj = vv[j >> 1] + 2 * (j & 1);
            adamw_one(pa, bf16_lo(g32[j]), mj[0], vj[0], lr, b1, b2, eps, wd, bc1, bc2_sqrt, decoupled);
            adamw_one(pb, bf16_hi(g32[j]), mj[1], vj[1], lr, b1, b2, eps, wd, bc1, bc2_sqrt, decoupled);
            p32[j] = pack_bf16(pa, pb);
        }
        if (STREAM) {
            __stcs(reinterpret_cast<uint4*>(p) + i, pu);
            __stcs(reinterpret_cast<float4*>(m) + 2 * i, m0); __stcs(reinterpret_cast<float4*>(m) + 2 * i + 1, m1);
            __stcs(reinterpret_cast<float4*>(v) + 2 * i, v0); __stcs(reinterpret_cast<float4*>(v) + 2 * i + 1, v1);
        } else {
            reinterpret_cast<uint4*>(p)[i] = pu;
            reinterpret_cast<float4*>(m)[2 * i] = m0; reinterpret_cast<float4*>(m)[2 * i + 1] = m1;
            reinterpret_cast<float4*>(v)[2 * i] = v0; reinterpret_cast<float4*>(v)[2 * i + 1] = v1;
        }
    }
    // tail (n % 8 elements)
    for (size_t i = (n8 << 3) + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        float pw = bf2f(p[i]), mi = m[i], vi = v[i];
        adamw_one(pw, bf2f(g[i]), mi, vi, lr, b1, b2, eps, wd, bc1, bc2_sqrt, decoupled);
        m[i] = mi; v[i] = vi; p[i] = f2bf(pw);
    }
}

// acc[c] += sum_b part[b * ld + c] for b = 0..nb-1 in order.  Kernels that reduce over rows write one partial row per
// CTA instead of adding with float atomics: atomics add in whatever order the CTAs finish, so two runs of one training
// step would differ in the last bits and, through the optimizer, drift apart.
__global__ void det_reduce_kernel(const float* __restrict__ part, int nb, int n, int ld, float* __restrict__ acc) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n) return;
    float s = 0.f;
    for (int b = 0; b < nb; ++b) s += part[(size_t)b * ld + c];
    acc[c] += s;
}

// stream-ordered scratch for the partial rows (the default memory pool keeps it cached)
static float* det_alloc(size_t floats, cudaStream_t st) {
    void* p = nullptr;
    if (cudaMallocAsync(&p, floats * sizeof(float), st) != cudaSuccess) {
        set_error("stream-ordered allocation of %zu bytes failed", floats * sizeof(float));
        return nullptr;
    }
    return (float*)p;
}
static int det_finish(float* part, int nb, int n, int ld, float* acc, cudaStream_t st, const char* what) {
    det_reduce_kernel<<<(n + 127) / 128, 128, 0, st>>>(part, nb, n, ld, acc);
    cudaFreeAsync(part, st);
    return check_launch(what);
}

static inline int ew_grid(size_t n, int threads) {
    size_t b = (n + threads - 1) / threads;
    const size_t cap = (size_t)sm_count() * 16;
    return (int)(b < cap ? (b ? b : 1) : cap);
}

}  // namespace tl

extern "C" {

int tl_swiglu_fwd(const void* gu, void* h, int M, int I, void* stream) {
    using namespace tl;
    TL_REQUIRE(I % 4 == 0, TL_ERR_INVALID, "tl_swiglu_fwd: I %% 4 != 0");
    const size_t n_vec = (size_t)M * I / 4;
    if (!n_vec) return TL_OK;
    swiglu_fwd_kernel<<<ew_grid(n_vec, 256), 256, 0, (cudaStream_t)stream>>>((const uint4*)gu, (uint2*)h, n_vec);
    return check_launch("tl_swiglu_fwd");
}

int tl_swiglu_bwd(const void* gu, const void* dh, void* dgu, int M, int I, void* stream) {
    using namespace tl;
    TL_REQUIRE(I % 4 == 0, TL_ERR_INVALID, "tl_swiglu_bwd: I %% 4 != 0");
    const size_t n_vec = (size_t)M * I / 4;
    if (!n_vec) return TL_OK;
    swiglu_bwd_kernel<<<ew_grid(n_vec, 256), 256, 0, (cudaStream_t)stream>>>((const uint4*)gu, (const uint2*)dh, (uint4*)dgu, n_vec);
    return check_launch("tl_swiglu_bwd");
}

int tl_rmsnorm_bwd(const void* x, const void* w, const void* dy, const float* rstd, const void* dx_add, void* dx,
                   float* dw_accum, int rows, int H, void* stream) {
    using namespace tl;
    TL_REQUIRE(H % 8 == 0 && H <= NB_THREADS * 8 * 8, TL_ERR_INVALID, "tl_rmsnorm_bwd: unsupported H=%d", H);
    if (rows == 0) return TL_OK;
    static int mult = 0;                       // CTAs per SM worth of row blocks (TL_NB_GRID_MULT, default 2)
    if (mult == 0) {
        const char* e = getenv("TL_NB_GRID_MULT");
        mult = e ? atoi(e) : 2;
        if (mult < 1 || mult > 16) mult = 2;
    }
    int rpb = (rows + sm_count() * mult - 1) / (sm_count() * mult);
    if (rpb < 1) rpb = 1;
    const int grid = (rows + rpb - 1) / rpb;
    const int nv = ((H >> 3) + NB_THREADS - 1) / NB_THREADS;
    cudaStream_t st = (cudaStream_t)stream;
    const bool warp_rows = (H >> 3) <= 32 * NBW_MAXV;
    int g = (rows + 3) / 4;
    if (g > sm_count() * 4) g = sm_count() * 4;
    const int nb = warp_rows ? g : grid;
    float* part = nullptr;
    if (dw_accum && !(part = det_alloc((size_t)nb * H, st))) return TL_ERR_CUDA;
    if (warp_rows) {
        rmsnorm_bwd_warp_kernel<<<g, NB_THREADS, 0, st>>>((const bf16*)x, (const bf16*)w, (const bf16*)dy, rstd,
                                                          (const bf16*)dx_add, (bf16*)dx, part, rows, H);
    } else {
#define TL_NB(MV)                                                                                                       \
    rmsnorm_bwd_kernel<MV><<<grid, NB_THREADS, 0, st>>>((const bf16*)x, (const bf16*)w, (const bf16*)dy, rstd,          \
                                                       (const bf16*)dx_add, (bf16*)dx, part, rows, H, rpb)
        if (nv <= 1) TL_NB(1);
        else if (nv <= 2) TL_NB(2);
        else if (nv <= 4) TL_NB(4);
        else TL_NB(8);
#undef TL_NB
    }
    if (!part) return check_launch("tl_rmsnorm_bwd");
    const int rc = check_launch("tl_rmsnorm_bwd");
    if (rc != TL_OK) { cudaFreeAsync(part, st); return rc; }
    return det_finish(part, nb, H, H, dw_accum, st, "tl_rmsnorm_bwd (dw reduce)");
}

int tl_rope_kv_bwd(const void* dq, const void* dk, const void* dv, void* dqkv, const void* cos_tab, const void* sin_tab,
                   int n_tokens, int S, int n_h, int n_kv, int d, int T_max, void* stream) {
    using namespace tl;
    TL_REQUIRE(d == 64 || d == 128, TL_ERR_INVALID, "tl_rope_kv_bwd: head_dim %d not in {64,128}", d);
    if (n_tokens == 0) return TL_OK;
    const long long warps = (long long)n_tokens * (n_h + 2 * n_kv);
    const int grid = (int)((warps + 3) / 4);
    cudaStream_t st = (cudaStream_t)stream;
    if (d == 64)
        rope_kv_bwd_kernel<64><<<grid, 128, 0, st>>>((const bf16*)dq, (const bf16*)dk, (const bf16*)dv, (bf16*)dqkv,
                                                     (const bf16*)cos_tab, (const bf16*)sin_tab, n_tokens, S, n_h, n_kv, T_max);
    else
        rope_kv_bwd_kernel<128><<<grid, 128, 0, st>>>((const bf16*)dq, (const bf16*)dk, (const bf16*)dv, (bf16*)dqkv,
                                                      (const bf16*)cos_tab, (const bf16*)sin_tab, n_tokens, S, n_h, n_kv, T_max);
    return check_launch("tl_rope_kv_bwd");
}

int tl_qk_norm_bwd(const void* qkv_pre, void* dqkv, const void* q_norm_w, const void* k_norm_w, float* dqn_accum,
                   float* dkn_accum, float eps, int n_tokens, int n_h, int n_kv, int d, void* stream) {
    using namespace tl;
    TL_REQUIRE(d == 64 || d == 128, TL_ERR_INVALID, "tl_qk_norm_bwd: head_dim %d not in {64,128}", d);
    if (n_tokens == 0) return TL_OK;
    const long long warps = (long long)n_tokens * (n_h + n_kv);
    long long g = (warps + 3) / 4;
    if (g > sm_count() * 4) g = sm_count() * 4;
    const int grid = (int)g;
    cudaStream_t st = (cudaStream_t)stream;
    float* part = det_alloc((size_t)grid * 2 * d, st);
    if (!part) return TL_ERR_CUDA;
    if (d == 64)
        qk_norm_bwd_kernel<64><<<grid, 128, 0, st>>>((const bf16*)qkv_pre, (bf16*)dqkv, (const bf16*)q_norm_w, (const bf16*)k_norm_w,
                                                     part, eps, n_tokens, n_h, n_kv);
    else
        qk_norm_bwd_kernel<128><<<grid, 128, 0, st>>>((const bf16*)qkv_pre, (bf16*)dqkv, (const bf16*)q_norm_w, (const bf16*)k_norm_w,
                                                      part, eps, n_tokens, n_h, n_kv);
    int rc = check_launch("tl_qk_norm_bwd");
    if (rc != TL_OK) { cudaFreeAsync(part, st); return rc; }
    det_reduce_kernel<<<(d + 127) / 128, 128, 0, st>>>(part + d, grid, d, 2 * d, dkn_accum);
    return det_finish(part, grid, d, 2 * d, dqn_accum, st, "tl_qk_norm_bwd (gain reduce)");   // frees part
}

int tl_ce_fwd_bwd(const void* logits, const int64_t* labels, float* loss_sum, int32_t* n_valid, void* dlogits,
                  float grad_scale, int M, int V, void* stream) {
    using namespace tl;
    TL_REQUIRE(V % 8 == 0, TL_ERR_INVALID, "tl_ce_fwd_bwd: V %% 8 != 0");
    if (M == 0) return TL_OK;
    cudaStream_t st = (cudaStream_t)stream;
    float* part = det_alloc((size_t)M, st);
    if (!part) return TL_ERR_CUDA;
    ce_fwd_bwd_kernel<<<M, CE_THREADS, 0, st>>>((const bf16*)logits, labels, part, n_valid, (bf16*)dlogits, grad_scale, V);
    const int rc = check_launch("tl_ce_fwd_bwd");
    if (rc != TL_OK) { cudaFreeAsync(part, st); return rc; }
    return det_finish(part, M, 1, 1, loss_sum, st, "tl_ce_fwd_bwd (loss reduce)");
}

int tl_embed_bwd(const int64_t* ids, const void* dout, void* dtable, int n_tokens, int H, int vocab, void* stream) {
    using namespace tl;
    TL_REQUIRE(H % 2 == 0, TL_ERR_INVALID, "tl_embed_bwd: H odd");
    if (n_tokens == 0) return TL_OK;
    embed_bwd_kernel<<<(n_tokens + 7) / 8, 256, 0, (cudaStream_t)stream>>>(ids, (const bf16*)dout, (bf16*)dtable, n_tokens, H, vocab);
    return check_launch("tl_embed_bwd");
}

int tl_colsum(const void* dy, float* db_accum, int M, int N, int ld, void* stream) {
    using namespace tl;
    TL_REQUIRE(N % 2 == 0 && ld % 2 == 0, TL_ERR_INVALID, "tl_colsum: N/ld must be even");
    if (M == 0) return TL_OK;
    const dim3 grid((N / 2 + 31) / 32, (M + 255) / 256), block(32, 8);
    cudaStream_t st = (cudaStream_t)stream;
    float* part = det_alloc((size_t)grid.y * N, st);
    if (!part) return TL_ERR_CUDA;
    colsum_kernel<<<grid, block, 0, st>>>((const bf16*)dy, part, M, N, ld);
    const int rc = check_launch("tl_colsum");
    if (rc != TL_OK) { cudaFreeAsync(part, st); return rc; }
    return det_finish(part, (int)grid.y, N, N, db_accum, st, "tl_colsum (reduce)");
}

int tl_f32_to_bf16_accum(const float* src, void* dst, size_t n, int accumulate, void* stream) {
    using namespace tl;
    if (!n) return TL_OK;
    f32_to_bf16_accum_kernel<<<ew_grid(n, 256), 256, 0, (cudaStream_t)stream>>>(src, (bf16*)dst, n, accumulate);
    return check_launch("tl_f32_to_bf16_accum");
}

int tl_add_inplace(void* a, const void* b, size_t n, void* stream) {
    using namespace tl;
    TL_REQUIRE(n % 8 == 0, TL_ERR_INVALID, "tl_add_inplace: n %% 8 != 0");
    if (!n) return TL_OK;
    add_inplace_kernel<<<ew_grid(n / 8, 256), 256, 0, (cudaStream_t)stream>>>((uint4*)a, (const uint4*)b, n / 8);
    return check_launch("tl_add_inplace");
}

int tl_scale_add_bf16(void* a, const void* b, float scale, int accumulate, size_t n, void* stream) {
    using namespace tl;
    TL_REQUIRE(n % 8 == 0, TL_ERR_INVALID, "tl_scale_add_bf16: n %% 8 != 0");
    TL_REQUIRE(((((uintptr_t)a) | ((uintptr_t)b)) & 15) == 0, TL_ERR_INVALID, "tl_scale_add_bf16: 16-byte alignment required");
    if (!n) return TL_OK;
    scale_add_bf16_kernel<<<ew_grid(n / 8, 256), 256, 0, (cudaStream_t)stream>>>((uint4*)a, (const uint4*)b, scale, accumulate, n / 8);
    return check_launch("tl_scale_add_bf16");
}

int tl_scale_add_f32(float* a, const float* b, float scale, int accumulate, size_t n, void* stream) {
    using namespace tl;
    if (!n) return TL_OK;
    scale_add_f32_kernel<<<ew_grid(n, 256), 256, 0, (cudaStream_t)stream>>>(a, b, scale, accumulate, n);
    return check_launch("tl_scale_add_f32");
}

int tl_adamw_step(void* param, const void* grad, float* exp_avg, float* exp_avg_sq, size_t n, float lr, float beta1,
                  float beta2, float eps, float weight_decay, int step, int decoupled, void* stream) {
    using namespace tl;
    TL_REQUIRE(step >= 1, TL_ERR_INVALID, "tl_adamw_step: step must start at 1");
    if (!n) return TL_OK;
    TL_REQUIRE(((((uintptr_t)param) | ((uintptr_t)grad) | ((uintptr_t)exp_avg) | ((uintptr_t)exp_avg_sq)) & 15) == 0, TL_ERR_INVALID,
               "tl_adamw_step: arenas must be 16-byte aligned");
    const float bc1 = 1.0f - powf(beta1, (float)step);
    const float bc2s = sqrtf(1.0f - powf(beta2, (float)step));
    // evict-first loads / stores (the arena is touched once per step); TL_ADAM_STREAM=0 = plain
    static int stream_hint = -1;
    if (stream_hint < 0) {
        const char* e = getenv("TL_ADAM_STREAM");
        stream_hint = (e && e[0] == '0') ? 0 : 1;
    }
    if (stream_hint)
        adamw_kernel<true><<<ew_grid((n + 7) / 8, 256), 256, 0, (cudaStream_t)stream>>>((bf16*)param, (const bf16*)grad, exp_avg, exp_avg_sq,
                                                                              n, lr, beta1, beta2, eps, weight_decay, bc1, bc2s, decoupled);
    else
        adamw_kernel<false><<<ew_grid((n + 7) / 8, 256), 256, 0, (cudaStream_t)stream>>>((bf16*)param, (const bf16*)grad, exp_avg, exp_avg_sq,
                                                                               n, lr, beta1, beta2, eps, weight_decay, bc1, bc2s, decoupled);
    return check_launch("tl_adamw_step");
}

}  // extern "C"
