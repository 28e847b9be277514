// FP8 weights -> bf16: out[n,k] = bf16(float(W[n,k]) * scales[n][k/128]), HF's Fp8Dequantize followed by the cast to
// the model dtype.  The GEMM paths (prefill, batched decode, long verify steps) run tl_gemm_bf16 over this scratch copy.
// HBM-bound: 1 byte read + 2 bytes written per weight; each thread converts 8 consecutive weights per step.
#include <cuda_fp8.h>

#include "common.cuh"

namespace tl {

__global__ void __launch_bounds__(256) dequant_fp8_kernel(const uint2* __restrict__ W, const float* __restrict__ scales,
                                                          uint4* __restrict__ out, int K, size_t n_vec) {
    const int vpr = K >> 3;                          // 8-weight vectors per row
    const int groups = K / TL_FP8_BLOCK;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += (size_t)gridDim.x * blockDim.x) {
        const size_t row = i / vpr;
        const int v = (int)(i - row * vpr);
        const float s = __ldg(scales + row * groups + (v >> 4));
        const uint2 w = __ldg(W + i);
        const uint32_t u[2] = {w.x, w.y};
        uint4 o;
        uint32_t* o32 = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const __half2_raw r = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(u[h] >> (16 * j)), __NV_E4M3);
                const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&r));
                o32[2 * h + j] = pack_bf16(f.x * s, f.y * s);
            }
        out[i] = o;
    }
}

}  // namespace tl

extern "C" int tl_dequant_fp8(const void* W, const float* scales, void* out, int N, int K, void* stream) {
    using namespace tl;
    TL_REQUIRE(N > 0 && K > 0 && K % TL_FP8_BLOCK == 0, TL_ERR_INVALID, "tl_dequant_fp8: need K %% %d == 0 (N=%d K=%d)",
               TL_FP8_BLOCK, N, K);
    TL_REQUIRE(W && scales && out && ((uintptr_t)W & 7) == 0 && ((uintptr_t)out & 15) == 0 && ((uintptr_t)scales & 3) == 0,
               TL_ERR_INVALID, "tl_dequant_fp8: W must be 8-byte, out 16-byte and scales 4-byte aligned");
    const size_t n_vec = (size_t)N * (K >> 3);
    size_t grid = (n_vec + 255) / 256;
    const size_t cap = (size_t)sm_count() * 8;
    if (grid > cap) grid = cap;
    dequant_fp8_kernel<<<(unsigned)grid, 256, 0, (cudaStream_t)stream>>>((const uint2*)W, scales, (uint4*)out, K, n_vec);
    return check_launch("tl_dequant_fp8");
}
