"""Qwen3-30B-A3B (``configs.QWEN3_30B_A3B``, bf16, weights drawn on the device, training=False) on one H100.

* greedy batch-1 decode: ms per token = (t(NEW) - t(1)) / (NEW - 1) from host clocks around whole generate calls that end
  in a device synchronise (captured graphs), against the HBM bound of the bytes one token reads: attention, router and
  the top_k picked experts of every layer plus the final norm and lm_head (6.08 GB; the embedding is a row lookup);
* batched decode at 8 and 32 rows (same method), and prefill of 8 x 512 tokens (one forward);
* the expert GEMV alone (CUDA events, gate/up and down launches at one row, layer 0's experts) in TB/s, and the grouped
  GEMM alone (gate/up and down at 8 x 512 tokens routed by random logits) in TFLOP/s.

Random router weights route almost uniformly, so every decode row touches k distinct experts and a batched step touches
nearly min(E, rows x k) of them; checkpoints with real routing were not measured.

    python tools/bench_moe.py [--rounds 3] [--out FILE]

Prints one JSON line, with the card's name, power limit and max SM clock read in the same run.
"""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from bench_prompt_lookup import _card  # noqa: E402

PROMPT, NEW = 32, 64
HBM_TBPS = 3.35          # H100 SXM data sheet


def _timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def _events(fn, n=50):
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n / 1e3


def token_bytes(cfg) -> int:
    """Bytes of weights one decode token reads (bf16): active parameters without the embedding table."""
    return 2 * (cfg.active_params() - cfg.vocab * cfg.hidden)


def decode(dm, B, rounds):
    from tensorlink_b200.ml.weights import synthetic_tokens
    ids = synthetic_tokens(dm.cfg, B, PROMPT)
    dm.generate(ids, max_new_tokens=NEW)
    dm.generate(ids, max_new_tokens=1)
    ms = []
    for _ in range(rounds):
        t1 = _timed(lambda: dm.generate(ids, max_new_tokens=1))
        tn = _timed(lambda: dm.generate(ids, max_new_tokens=NEW))
        ms.append((tn - t1) / (NEW - 1) * 1e3)
    return statistics.median(ms), min(ms), max(ms)


def kernels(dm):
    from tensorlink_b200 import native as nat
    cfg, v = dm.cfg, dm.stage.params.v
    E, k, H, I = cfg.n_experts, cfg.top_k, cfg.hidden, cfg.moe_intermediate
    dev = "cuda"
    res = {}
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(1, H, device=dev, generator=g).bfloat16()
    ids = torch.randperm(E, device=dev, generator=g)[:k].sort().values.to(torch.int32).view(1, k)
    wts = torch.full((1, k), 1.0 / k, device=dev)
    act = torch.empty(k, I, device=dev).bfloat16()
    out = torch.empty(1, H, device=dev).bfloat16()
    t = _events(lambda: nat.moe_gemv(x, v["l0.ewgu"], act, ids, flags=nat.EPI_SWIGLU))
    res["gemv_gate_up"] = {"us": t * 1e6, "TBps": k * 2 * I * H * 2 / t / 1e12}
    t = _events(lambda: nat.moe_gemv(act, v["l0.ewd"], out, ids, wts=wts, residual=x, flags=nat.EPI_RESIDUAL))
    res["gemv_down"] = {"us": t * 1e6, "TBps": k * H * I * 2 / t / 1e12}
    N = 8 * 512
    logits = torch.randn(N, E, device=dev, generator=g).bfloat16()
    T = nat.moe_max_tiles(N, E, k)
    i32 = dict(dtype=torch.int32, device=dev)
    rid, rw = torch.empty(N, k, **i32), torch.empty(N, k, dtype=torch.float32, device=dev)
    plan = (torch.empty(E, **i32), torch.empty(E + 1, **i32), torch.empty(N * k, **i32), torch.empty(T, 2, **i32))
    nat.moe_route(logits, k, True, rid, rw, plan)
    h = torch.randn(N, H, device=dev, generator=g).bfloat16()
    hg = torch.empty(T * 128, H, device=dev).bfloat16()
    nat.moe_gather(h, plan[2], hg, k)
    a = torch.empty(T * 128, I, device=dev).bfloat16()
    y = torch.empty(T * 128, H, device=dev).bfloat16()
    t = _events(lambda: nat.moe_gemm(hg, v["l0.ewgu"], a, plan[3], flags=nat.EPI_SWIGLU), 20)
    res["grouped_gate_up"] = {"us": t * 1e6, "TFLOPs": 2 * N * k * 2 * I * H / t / 1e12}
    t = _events(lambda: nat.moe_gemm(a, v["l0.ewd"], y, plan[3]), 20)
    res["grouped_down"] = {"us": t * 1e6, "TFLOPs": 2 * N * k * H * I / t / 1e12}
    t = _events(lambda: nat.moe_route(logits, k, True, rid, rw, plan), 20)
    res["route_plan_8x512"] = {"us": t * 1e6}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from tensorlink_b200.ml import DistributedModel
    from tensorlink_b200.ml import configs as C
    from tensorlink_b200.ml.weights import synthetic_tokens
    cfg = C.QWEN3_30B_A3B
    dm = DistributedModel(cfg, training=False, max_batch=32, max_seq=640, init="device")
    res = {"model": cfg.name, "card": _card(), "token_bytes_GB": token_bytes(cfg) / 1e9,
           "note": "random router weights route almost uniformly; routing of real checkpoints is not measured"}
    bound_ms = token_bytes(cfg) / (HBM_TBPS * 1e12) * 1e3
    for B in (1, 8, 32):
        med, lo, hi = decode(dm, B, a.rounds)
        r = {"ms_per_step": med, "range": [lo, hi], "tokens_per_s": B * 1e3 / med}
        if B == 1:
            r["hbm_bound_ms"] = bound_ms
            r["frac_of_hbm_bound"] = bound_ms / med
        res[f"decode_B{B}"] = r
    ids = synthetic_tokens(cfg, 8, 512)
    dm(ids)
    ts = [_timed(lambda: dm(ids)) for _ in range(a.rounds)]
    res["prefill_8x512"] = {"s": statistics.median(ts), "tokens_per_s": 8 * 512 / statistics.median(ts)}
    res["kernels"] = kernels(dm)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
