// FP8 weights (HF's fine-grained float8_e4m3fn, one fp32 scale per row and 128 columns) for the GEMV kernels.
#pragma once
#include <cuda_fp8.h>

#include "common.cuh"

namespace tl {

typedef __nv_fp8_e4m3 fp8_e4m3;

// 8 consecutive FP8 weights of one row -> bf16(float(w) * scale), as floats.  e4m3 -> f16 is exact.
__device__ __forceinline__ void fp8x8_scaled(uint2 w, float scale, float (&f)[8]) {
    const uint32_t u[2] = {w.x, w.y};
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const __half2_raw r = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(u[h] >> (16 * j)), __NV_E4M3);
            const float2 v = __half22float2(*reinterpret_cast<const __half2*>(&r));
            f[4 * h + 2 * j] = rbf(v.x * scale);
            f[4 * h + 2 * j + 1] = rbf(v.y * scale);
        }
}

}  // namespace tl
