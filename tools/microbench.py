"""Kernel micro-benchmarks on one H100 (CUDA events, rotating buffers larger than L2).  Not a bench line."""
import json
import sys
import os

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tensorlink_b200 import native as nat  # noqa: E402


def timeit(fn, n_rot, iters=20, warm=5):
    for i in range(warm):
        fn(i % n_rot)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fn(i % n_rot)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e-3


def bench_gemv(M, N, K, flags=0, norm=False):
    n_rot = max(2, int(300e6 // (N * K * 2)) + 1)
    ws = [torch.randn(N, K, device="cuda").bfloat16() * 0.05 for _ in range(n_rot)]
    x = torch.randn(M, K, device="cuda").bfloat16()
    g = torch.ones(K, device="cuda").bfloat16() if norm else None
    out = torch.empty(M, N // 2 if flags & nat.EPI_SWIGLU else N, device="cuda", dtype=torch.bfloat16)
    t = timeit(lambda i: nat.gemv(x, ws[i], out, norm_w=g, flags=flags), n_rot)
    return {"op": "gemv", "M": M, "N": N, "K": K, "us": t * 1e6, "GBps": N * K * 2 / t / 1e9}


def bench_gemm(M, N, K, flags=0):
    n_rot = 2
    a = [torch.randn(M, K, device="cuda").bfloat16() for _ in range(n_rot)]
    w = [torch.randn(N, K, device="cuda").bfloat16() * 0.05 for _ in range(n_rot)]
    out = torch.empty(M, N // 2 if flags & nat.EPI_SWIGLU else N, device="cuda", dtype=torch.bfloat16)
    t = timeit(lambda i: nat.gemm(a[i], w[i], out, flags=flags), n_rot)
    tc = timeit(lambda i: torch.matmul(a[i], w[i].t()), n_rot)
    return {"op": "gemm", "M": M, "N": N, "K": K, "us": t * 1e6, "TFLOPs": 2 * M * N * K / t / 1e12,
            "cublas_TFLOPs": 2 * M * N * K / tc / 1e12}


def main():
    nat.require_device()
    res = []
    for (M, N, K, fl, nm) in [(1, 4608, 3584, 0, True), (1, 3584, 3584, 0, False), (1, 37888, 3584, nat.EPI_SWIGLU, True),
                              (1, 3584, 18944, 0, False), (1, 152064, 3584, 0, True), (4, 37888, 3584, nat.EPI_SWIGLU, True),
                              (1, 1152, 896, 0, True), (1, 9728, 896, nat.EPI_SWIGLU, True), (1, 896, 4864, 0, False),
                              (1, 151936, 896, 0, True), (2, 37888, 3584, nat.EPI_SWIGLU, True), (8, 37888, 3584, nat.EPI_SWIGLU, True),
                              (4, 3584, 18944, 0, False), (8, 3584, 18944, 0, False), (8, 4608, 3584, 0, True)]:
        r = bench_gemv(M, N, K, fl, nm)
        print(json.dumps(r), flush=True)
        res.append(r)
    for (M, N, K, fl) in [(4096, 4608, 3584, 0), (4096, 3584, 3584, 0), (4096, 37888, 3584, nat.EPI_SWIGLU),
                          (4096, 3584, 18944, 0), (8192, 8192, 8192, 0), (2048, 4608, 3584, 0), (4096, 1152, 896, 0),
                          (4096, 9728, 896, nat.EPI_SWIGLU), (4096, 896, 4864, 0), (32, 37888, 3584, nat.EPI_SWIGLU)]:
        r = bench_gemm(M, N, K, fl)
        print(json.dumps(r), flush=True)
        res.append(r)
    os.makedirs("gpurun_out", exist_ok=True)
    json.dump(res, open("gpurun_out/microbench.json", "w"), indent=1)


if __name__ == "__main__":
    main()
