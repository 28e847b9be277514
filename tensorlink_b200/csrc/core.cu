// Error plumbing, device probing, tiny device-side helpers.
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

namespace tl {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("%s: %s", what, cudaGetErrorString(e));
        return TL_ERR_CUDA;
    }
    return TL_OK;
}

int sm_count() {
    static int cached = 0;
    if (cached == 0) {
        int dev = 0, n = 0;
        if (cudaGetDevice(&dev) != cudaSuccess ||
            cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
            cudaGetLastError();
            return 132;
        }
        cached = n;
    }
    return cached;
}

__global__ void advance_pos_kernel(int32_t* pos, int32_t* kv_len, int delta) {
    int p = *pos + delta;
    *pos = p;
    if (kv_len) *kv_len = p;
}

// out_tokens[b, *step] = ids[b]; then ++*step  (one thread block, B <= 1024)
__global__ void append_token_kernel(const int64_t* ids, int64_t* out_tokens, int32_t* step, int B, int ld) {
    const int s = *step;
    __syncthreads();
    if ((int)threadIdx.x < B && s < ld) out_tokens[(size_t)threadIdx.x * ld + s] = ids[threadIdx.x];
    if (threadIdx.x == 0) *step = s + 1;
}

}  // namespace tl

extern "C" {

int tl_abi_version(void) { return TL_ABI_VERSION; }

const char* tl_last_error(void) { return tl::g_err; }

int tl_device_info(int* sm_count, int* cc_major, int* cc_minor) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
        cudaGetLastError();
        tl::set_error("no CUDA device visible; tensorlink_b200 has no CPU path");
        return TL_ERR_NO_DEVICE;
    }
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceProp p;
    if (cudaGetDeviceProperties(&p, dev) != cudaSuccess) {
        tl::set_error("cudaGetDeviceProperties failed");
        return TL_ERR_CUDA;
    }
    if (sm_count) *sm_count = p.multiProcessorCount;
    if (cc_major) *cc_major = p.major;
    if (cc_minor) *cc_minor = p.minor;
    if (p.major != 9 || p.minor != 0) {
        tl::set_error("device is sm_%d%d; this library is built for sm_90a (H100) only", p.major, p.minor);
        return TL_ERR_NO_DEVICE;
    }
    return TL_OK;
}

int tl_advance_pos(int32_t* pos_dev, int32_t* kv_len_dev, int delta, void* stream) {
    TL_REQUIRE(pos_dev != nullptr, TL_ERR_INVALID, "tl_advance_pos: null pos");
    tl::advance_pos_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(pos_dev, kv_len_dev, delta);
    return tl::check_launch("tl_advance_pos");
}

int tl_append_token(const int64_t* ids, int64_t* out_tokens, int32_t* step_dev, int B, int ld, void* stream) {
    TL_REQUIRE(ids && out_tokens && step_dev && B >= 1 && B <= 1024, TL_ERR_INVALID, "tl_append_token: bad args");
    tl::append_token_kernel<<<1, ((B + 31) / 32) * 32, 0, (cudaStream_t)stream>>>(ids, out_tokens, step_dev, B, ld);
    return tl::check_launch("tl_append_token");
}

}  // extern "C"
