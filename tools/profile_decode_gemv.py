"""Where a batch-1 decode step's time goes, per weight-streaming GEMV shape, against a streaming ceiling measured in the
same run.

    python tools/profile_decode_gemv.py [--model Qwen/Qwen2.5-7B] [--prompt 32] [--new 32] [--json OUT]

On the bench workload (greedy generate, one row, captured decode graphs) it reports
  * the decode step time (CUDA events around the token loop, profiler off);
  * from torch.profiler, every ``gemv_stream_kernel`` launch of the decode steps, grouped by shape (qkv, o, gate/up,
    down, lm_head): mean duration and achieved GB/s (algorithmic bytes 2*N*K over the duration), and the same over
    the exclusive part of the duration (after the kernels launched before it ended: the overlap that programmatic
    dependent launch allows is counted once);
  * the summed duration of all kernels of the decode steps against the step time (launches overlap under programmatic
    dependent launch, so the sum can exceed the step);
  * a read-only streaming ceiling: a 2 GiB buffer read with 16-byte vector loads by a probe kernel compiled at run
    time into a temporary directory, best of several passes;
  * the card name, power limit and maximum SM clock.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tensorlink_b200.ml import DistributedModel  # noqa: E402
from tensorlink_b200.ml.configs import get_config  # noqa: E402
from tensorlink_b200.ml.weights import synthetic_tokens  # noqa: E402

PROBE_SRC = r"""
#include <cstdint>
extern "C" __global__ void __launch_bounds__(512) read_probe(const uint4* __restrict__ p, size_t n, unsigned* sink) {
    unsigned acc = 0;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (; i + 3 * stride < n; i += 4 * stride) {
        const uint4 a = __ldg(p + i), b = __ldg(p + i + stride), c = __ldg(p + i + 2 * stride), d = __ldg(p + i + 3 * stride);
        acc ^= a.x ^ a.y ^ a.z ^ a.w ^ b.x ^ b.y ^ b.z ^ b.w ^ c.x ^ c.y ^ c.z ^ c.w ^ d.x ^ d.y ^ d.z ^ d.w;
    }
    for (; i < n; i += stride) {
        const uint4 a = __ldg(p + i);
        acc ^= a.x ^ a.y ^ a.z ^ a.w;
    }
    if (acc == 0x9e3779b9u) atomicAdd(sink, 1u);      // keeps the loads alive; practically never taken
}
extern "C" int launch_read_probe(const void* p, size_t n_vec, unsigned* sink, int grid, void* stream) {
    read_probe<<<grid, 512, 0, (cudaStream_t)stream>>>((const uint4*)p, n_vec, sink);
    return (int)cudaGetLastError();
}
"""


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clk = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "sm_clock_max": clk}
    except (OSError, ValueError, subprocess.SubprocessError):
        return {"name": torch.cuda.get_device_name(), "power_limit": "unknown", "sm_clock_max": "unknown"}


def read_ceiling(gib=2.0, passes=10):
    """GB/s of the best of ``passes`` reads of a ``gib`` GiB device buffer (16-byte loads, 4 in flight per thread)."""
    tmp = tempfile.mkdtemp(prefix="tl_probe_")
    src, lib = os.path.join(tmp, "probe.cu"), os.path.join(tmp, "probe.so")
    with open(src, "w") as f:
        f.write(PROBE_SRC)
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    subprocess.run([nvcc if os.path.exists(nvcc) else "nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3",
                    "-shared", "-Xcompiler", "-fPIC", "-o", lib, src], check=True)
    so = ctypes.CDLL(lib)
    so.launch_read_probe.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    n_bytes = int(gib * (1 << 30))
    buf = torch.randn(n_bytes // 2, device="cuda").to(torch.bfloat16)
    sink = torch.zeros(1, dtype=torch.int32, device="cuda")
    grid = torch.cuda.get_device_properties(0).multi_processor_count * 4
    stream = torch.cuda.current_stream().cuda_stream

    def once():
        rc = so.launch_read_probe(buf.data_ptr(), n_bytes // 16, sink.data_ptr(), grid, stream)
        assert rc == 0, rc
    once()
    best = 0.0
    for _ in range(passes):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); once(); e1.record()
        torch.cuda.synchronize()
        best = max(best, n_bytes / (e0.elapsed_time(e1) * 1e-3) / 1e9)
    del buf
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="Qwen/Qwen2.5-7B")
    ap.add_argument("--prompt", type=int, default=32)
    ap.add_argument("--new", type=int, default=32)
    ap.add_argument("--json", default=None, help="also write the result to this file")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    cfg = get_config(a.model)
    dm = DistributedModel(a.model, training=False, max_batch=1, max_seq=a.prompt + a.new + 8, init="device",
                          max_tokens=a.prompt)
    ids = synthetic_tokens(cfg, 1, a.prompt).cuda()
    for _ in range(3):
        dm.generate(ids, max_new_tokens=a.new)
    torch.cuda.synchronize()
    spans = []
    for _ in range(5):
        dm.generate(ids, max_new_tokens=a.new, profile=True)
        spans.append(dm.timers["decode_span_s"] / (a.new - 1))
    spans.sort()
    step_s = spans[len(spans) // 2]

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        dm.generate(ids, max_new_tokens=a.new)
        torch.cuda.synchronize()
    kern = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and e.time_range.elapsed_us() > 0),
                  key=lambda e: e.time_range.start)
    gemv = [e for e in kern if "gemv_stream_kernel" in e.name]
    L = cfg.n_layers
    per_step = 4 * L + 1                      # qkv, o, gate/up, down per layer, then the lm_head
    n_dec = a.new - 1
    dec = gemv[-n_dec * per_step:]
    assert len(dec) == n_dec * per_step, (len(gemv), per_step)
    names = ("qkv", "o", "gate_up", "down")
    byts = {"qkv": 2 * cfg.qkv_dim * cfg.hidden, "o": 2 * cfg.hidden * cfg.q_dim, "gate_up": 4 * cfg.intermediate * cfg.hidden,
            "down": 2 * cfg.hidden * cfg.intermediate, "lm_head": 2 * cfg.vocab * cfg.hidden}
    # a kernel launched with programmatic dependent launch starts while its predecessor still runs: its duration
    # includes that overlap.  "exclusive" counts only the part after every kernel that started before it had ended.
    excl, horizon = {}, 0.0
    for e in kern:
        excl[id(e)] = max(0.0, e.time_range.end - max(e.time_range.start, horizon)) * 1e-6
        horizon = max(horizon, e.time_range.end)
    dur = {k: [] for k in byts}
    dur_x = {k: [] for k in byts}
    for i, e in enumerate(dec):
        j = i % per_step
        k = "lm_head" if j == 4 * L else names[j % 4]
        dur[k].append(e.time_range.elapsed_us() * 1e-6)
        dur_x[k].append(excl[id(e)])
    t0, t1 = dec[0].time_range.start, dec[-1].time_range.end
    in_window = [e for e in kern if e.time_range.start >= t0 and e.time_range.end <= t1]
    sum_kernels_s = sum(e.time_range.elapsed_us() for e in in_window) * 1e-6 / n_dec
    ceiling = read_ceiling()
    shapes = {}
    gemv_s = gemv_b = 0.0
    for k, ts in dur.items():
        t = sum(ts) / len(ts)
        tx = sum(dur_x[k]) / len(ts)
        n_per = 1 if k == "lm_head" else L
        gemv_s += t * n_per
        gemv_b += byts[k] * n_per
        shapes[k] = {"bytes": byts[k], "launches_per_step": n_per, "us": t * 1e6, "GBps": byts[k] / t / 1e9,
                     "frac_of_ceiling": byts[k] / t / 1e9 / ceiling, "us_exclusive": tx * 1e6,
                     "GBps_exclusive": byts[k] / tx / 1e9 if tx else None}
    res = {"model": a.model, "card": card(), "read_ceiling_GBps": ceiling, "step_ms": step_s * 1e3,
           "gemv_ms_per_step": gemv_s * 1e3, "gemv_GBps": gemv_b / gemv_s / 1e9, "gemv_frac_of_ceiling": gemv_b / gemv_s / 1e9 / ceiling,
           "all_kernels_ms_per_step": sum_kernels_s * 1e3, "shapes": shapes}
    print(json.dumps(res, indent=1))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
