// Shared pieces of the wgmma kernels (gemm.cu, attention_wgmma.cu): tensor-map construction, the wgmma / shared-memory descriptor PTX, and the
// accumulator -> registers -> shared-memory staging -> HBM epilogue.
//
// Epilogue layout.  The epilogue hands every thread of a warp ONE accumulator row (read back from the fp32 staging tile),
// so a direct store would make each warp instruction touch 32 different rows (32 partial sectors, row pitch = N*2 bytes
// apart).  Instead a warp stages its 32 rows x 64 columns through a private 32 x 144-byte shared-memory tile and then
// writes (and, for the residual / accumulate operands, reads) global memory with 8 lanes per row: every instruction moves
// four complete 128-byte lines.  Both shared-memory access patterns (row-per-lane and 8-lanes-per-row) are bank-conflict
// free with the 144-byte pitch.
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace tl {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int EPI_PITCH = 144;                       // bytes per staged row (128 + 16 pad)
constexpr int EPI_STAGE_BYTES = 32 * EPI_PITCH;      // per epilogue warp
constexpr int EPI_SMEM_BYTES = 4 * EPI_STAGE_BYTES;  // four epilogue warps

// ---------------------------------------------------------------------------------------- wgmma (sm_90a)
// Hopper shared-memory matrix descriptor: [0,14) start>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [49,52) base offset (0: tiles
// are 1024-byte aligned) | [62,64) layout (1 = SWIZZLE_128B, the layout TMA writes with CU_TENSOR_MAP_SWIZZLE_128B).
__device__ __forceinline__ uint64_t make_wgmma_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an asynchronous wgmma
template <int R>
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, both operands in shared memory; TA / TB = 1: operand is MN-major.
// Accumulator fragment: register i of thread (warp w, lane l) holds row 16w + l/4 + 8*((i>>1)&1), column 8*(i>>2) + 2*(l&3) + (i&1).
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n32(float (&d)[16], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

// A from registers: a[0..3] = the m64k16 A fragment of this thread (same layout as an m64n16 accumulator, packed bf16x2)
template <int TB>
__device__ __forceinline__ void wgmma_rs_m64n64(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1, %38;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d), "n"(TB));
}

// A from registers: a[0..3] = the m64k16 A fragment of this thread (same layout as an m64n16 accumulator, packed bf16x2)
template <int TB>
__device__ __forceinline__ void wgmma_rs_m64n128(float (&d)[64], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1, %70;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d), "n"(TB));
}

// 2-D bf16 row-major tensor [outer, inner] with leading dimension ld (elements); 128B-swizzled boxes (cached)
int make_tensor_map(CUtensorMap* out, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_inner,
                    uint32_t box_outer);

// coalesced [32 rows x 128 bytes] global -> staging tile (rows beyond M / pieces beyond `valid_bytes` read as zero)
__device__ __forceinline__ void epi_load_tile(unsigned char* stg, const unsigned char* gbase, size_t row_pitch_bytes, int row0,
                                              int M, int valid_bytes, int lane) {
    const int piece = lane & 7;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int rr = i * 4 + (lane >> 3);
        uint4 v = make_uint4(0, 0, 0, 0);
        if (row0 + rr < M && piece * 16 < valid_bytes)
            v = *reinterpret_cast<const uint4*>(gbase + (size_t)rr * row_pitch_bytes + piece * 16);
        *reinterpret_cast<uint4*>(stg + rr * EPI_PITCH + piece * 16) = v;
    }
    __syncwarp();
}
// staging tile -> coalesced global store of `row_bytes` (64 or 128) per row
__device__ __forceinline__ void epi_store_tile(const unsigned char* stg, unsigned char* gbase, size_t row_pitch_bytes, int row0,
                                               int M, int row_bytes, int valid_bytes, int lane) {
    __syncwarp();
    if (row_bytes == 128) {
        const int piece = lane & 7;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int rr = i * 4 + (lane >> 3);
            if (row0 + rr < M && piece * 16 < valid_bytes)
                *reinterpret_cast<uint4*>(gbase + (size_t)rr * row_pitch_bytes + piece * 16) =
                    *reinterpret_cast<const uint4*>(stg + rr * EPI_PITCH + piece * 16);
        }
    } else {   // 64 bytes per row: 4 lanes per row, 8 rows per instruction
        const int piece = lane & 3;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int rr = i * 8 + (lane >> 2);
            if (row0 + rr < M && piece * 16 < valid_bytes)
                *reinterpret_cast<uint4*>(gbase + (size_t)rr * row_pitch_bytes + piece * 16) =
                    *reinterpret_cast<const uint4*>(stg + rr * EPI_PITCH + piece * 16);
        }
    }
    __syncwarp();
}

// One 64-column chunk of one epilogue warp: r0 / r1 = fp32 accumulators of this thread's row for columns
// [col0, col0+32) and [col0+32, col0+64).  row0 = first row of the warp (thread `lane` owns row0 + lane).
__device__ __forceinline__ void gemm_epilogue_chunk64(const uint32_t (&r0)[32], const uint32_t (&r1)[32], unsigned char* stg,
                                                      void* Cv, int row0, int lane, int col0, int M, int N, int ldc,
                                                      const bf16* __restrict__ bias, const bf16* __restrict__ residual,
                                                      int ldr, int flags, int max_cols = 64) {
    if (row0 >= M || col0 >= N) return;                 // warp-uniform
    const int ncols = min(max_cols, N - col0);          // multiple of 8 (max_cols = 32 for 32-wide tiles)
    float v[64];
#pragma unroll
    for (int j = 0; j < 32; ++j) {
        v[j] = __uint_as_float(r0[j]);
        v[32 + j] = __uint_as_float(r1[j]);
    }
    if (flags & TL_EPI_BIAS) {
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            if (q * 8 < ncols) {
                const uint4 b4 = *reinterpret_cast<const uint4*>(bias + col0 + q * 8);
                const uint32_t* b32 = reinterpret_cast<const uint32_t*>(&b4);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    v[q * 8 + 2 * j] += bf16_lo(b32[j]);
                    v[q * 8 + 2 * j + 1] += bf16_hi(b32[j]);
                }
            }
        }
    }
    unsigned char* myrow = stg + lane * EPI_PITCH;
    if (flags & TL_EPI_SWIGLU) {
        // interleaved (gate, up) column pairs -> 32 bf16 outputs (64 bytes) per row
        uint32_t o[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const float g0 = rbf(v[4 * j]), u0 = rbf(v[4 * j + 1]);
            const float g1 = rbf(v[4 * j + 2]), u1 = rbf(v[4 * j + 3]);
            o[j] = pack_bf16(rbf(silu_f(g0)) * u0, rbf(silu_f(g1)) * u1);
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) *reinterpret_cast<uint4*>(myrow + q * 16) = make_uint4(o[4 * q], o[4 * q + 1], o[4 * q + 2], o[4 * q + 3]);
        unsigned char* g = reinterpret_cast<unsigned char*>(Cv) + ((size_t)row0 * ldc + (col0 >> 1)) * 2;
        epi_store_tile(stg, g, (size_t)ldc * 2, row0, M, 64, ncols, lane);
        return;
    }
    if (flags & TL_EPI_OUT_F32) {
        // fp32 output: two half-chunks of 32 columns (128 bytes per row each)
#pragma unroll
        for (int hb = 0; hb < 2; ++hb) {
            const int c0 = col0 + hb * 32;
            if (c0 >= N || hb * 32 >= max_cols) break;
            const int vb = min(32, N - c0) * 4;
            unsigned char* g = reinterpret_cast<unsigned char*>(Cv) + ((size_t)row0 * ldc + c0) * 4;
            if (flags & TL_EPI_ACCUM) {
                epi_load_tile(stg, g, (size_t)ldc * 4, row0, M, vb, lane);
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const float4 o = *reinterpret_cast<const float4*>(myrow + q * 16);
                    v[hb * 32 + 4 * q] += o.x; v[hb * 32 + 4 * q + 1] += o.y; v[hb * 32 + 4 * q + 2] += o.z; v[hb * 32 + 4 * q + 3] += o.w;
                }
                __syncwarp();
            }
#pragma unroll
            for (int q = 0; q < 8; ++q)
                *reinterpret_cast<float4*>(myrow + q * 16) =
                    make_float4(v[hb * 32 + 4 * q], v[hb * 32 + 4 * q + 1], v[hb * 32 + 4 * q + 2], v[hb * 32 + 4 * q + 3]);
            epi_store_tile(stg, g, (size_t)ldc * 4, row0, M, 128, vb, lane);
        }
        return;
    }
    // bf16 output: the Linear's own rounding, then the optional residual / accumulate adds (each rounded like torch)
#pragma unroll
    for (int j = 0; j < 64; ++j) v[j] = rbf(v[j]);
    unsigned char* g = reinterpret_cast<unsigned char*>(Cv) + ((size_t)row0 * ldc + col0) * 2;
    if (flags & TL_EPI_RESIDUAL) {
        const unsigned char* rg = reinterpret_cast<const unsigned char*>(residual) + ((size_t)row0 * ldr + col0) * 2;
        epi_load_tile(stg, rg, (size_t)ldr * 2, row0, M, ncols * 2, lane);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const uint4 u = *reinterpret_cast<const uint4*>(myrow + q * 16);
            const uint32_t* u32 = reinterpret_cast<const uint32_t*>(&u);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                v[8 * q + 2 * j] += bf16_lo(u32[j]);
                v[8 * q + 2 * j + 1] += bf16_hi(u32[j]);
            }
        }
        __syncwarp();
    }
    if (flags & TL_EPI_ACCUM) {
        epi_load_tile(stg, g, (size_t)ldc * 2, row0, M, ncols * 2, lane);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const uint4 u = *reinterpret_cast<const uint4*>(myrow + q * 16);
            const uint32_t* u32 = reinterpret_cast<const uint32_t*>(&u);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                v[8 * q + 2 * j] += bf16_lo(u32[j]);
                v[8 * q + 2 * j + 1] += bf16_hi(u32[j]);
            }
        }
        __syncwarp();
    }
#pragma unroll
    for (int q = 0; q < 8; ++q)
        *reinterpret_cast<uint4*>(myrow + q * 16) =
            make_uint4(pack_bf16(v[8 * q], v[8 * q + 1]), pack_bf16(v[8 * q + 2], v[8 * q + 3]),
                       pack_bf16(v[8 * q + 4], v[8 * q + 5]), pack_bf16(v[8 * q + 6], v[8 * q + 7]));
    epi_store_tile(stg, g, (size_t)ldc * 2, row0, M, 128, ncols * 2, lane);
}

}  // namespace tl
