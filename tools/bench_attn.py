#!/usr/bin/env python
"""Prefill attention forward and backward alone: the mma.sync kernels vs the wgmma kernels, CUDA events, TFLOP/s.

    python tools/bench_attn.py
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tensorlink_b200 import native as nat  # noqa: E402

SHAPES = [(8, 512, 28, 4, 128), (1, 2048, 28, 4, 128), (1, 4096, 32, 8, 128), (8, 512, 14, 2, 64)]


def timed(fn, reps=20):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3 / reps


def main():
    torch.cuda.set_device(0)
    print(torch.cuda.get_device_name(0))
    for B, S, n_h, n_kv, d in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(0)
        q = torch.randn(B, S, n_h * d, device="cuda", generator=g).bfloat16()
        kc = torch.randn(B, n_kv, S, d, device="cuda", generator=g).bfloat16()
        vc = torch.randn(B, n_kv, S, d, device="cuda", generator=g).bfloat16()
        do = torch.randn(B, S, n_h * d, device="cuda", generator=g).bfloat16()
        out = torch.empty_like(q)
        lse = torch.empty(B, n_h, S, device="cuda")
        dq = torch.empty(B, S, n_h, d, dtype=torch.bfloat16, device="cuda")
        dk = torch.empty(B, n_h, S, d, dtype=torch.bfloat16, device="cuda")
        dv = torch.empty_like(dk)
        ws = torch.empty(nat.attn_bwd_ws(B, S, n_h), dtype=torch.uint8, device="cuda")
        flops = 2 * B * n_h * S * S * d          # causal: half of 4·B·n_h·S²·d
        row = [f"B={B} S={S} heads={n_h}/{n_kv} d={d}"]
        for impl in ("mma", "wgmma"):
            os.environ["TL_ATTN_IMPL"] = os.environ["TL_ATTN_BWD"] = impl
            tf = timed(lambda: nat.attn_prefill_fwd(q, kc, vc, out, lse, B, S, 0, n_h, n_kv, d, d ** -0.5))
            tb = timed(lambda: nat.attn_bwd(q, kc, vc, out, do, lse, dq, dk, dv, ws, B, S, n_h, n_kv, d, d ** -0.5))
            row.append(f"{impl}: fwd {flops / tf / 1e12:.0f} bwd {2.5 * flops / tb / 1e12:.0f} TFLOP/s")
        print(" | ".join(row))


if __name__ == "__main__":
    main()
