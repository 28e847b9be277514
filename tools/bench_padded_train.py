"""Training on a padded batch: one optimizer step (forward + backward + Adam through ``DistributedModel``) on a batch of
eight rows with eight real lengths from 64 to 512, left-padded and right-padded to S = 512, against a dense 8 x 512
batch.  The three versions alternate in one process; each reports samples/s and real (non-pad) tokens/s, median over
the rounds.  Then the attention backward alone, CUDA events, on the model's attention shape (heads, kv heads, head
dim) with the same left padding: ``tl_attn_bwd_rows`` against ``tl_attn_bwd`` on the same tensors.

    python tools/bench_padded_train.py [--model Qwen/Qwen2.5-0.5B] [--rounds 5] [--steps 5] [--out FILE]

Pad tokens still go through every Linear (no unpadding), so the GEMM time of a padded step stays at the dense level;
the left-padded attention skips its pad tiles.  Weights are synthetic (seeded): the timing does not depend on their
values.  Prints one JSON line, with the card name and power limit read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

LENGTHS = (64, 128, 192, 256, 320, 384, 448, 512)
S = 512


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def batches(cfg):
    B = len(LENGTHS)
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(0, cfg.vocab, (B, S), generator=g)
    left = torch.zeros(B, S, dtype=torch.int64)
    right = torch.zeros_like(left)
    for b, L in enumerate(LENGTHS):
        left[b, S - L:] = 1
        right[b, :L] = 1
    return {"left": (ids, left, ids.masked_fill(left == 0, -100)),
            "right": (ids, right, ids.masked_fill(right == 0, -100)),
            "dense": (ids, None, ids)}


def bench_step(name, rounds, steps):
    from tensorlink_b200.ml import DistributedModel
    from tensorlink_b200.ml import configs as C
    cfg = C.get_config(name)
    B = len(LENGTHS)
    dm = DistributedModel(name, training=True, max_batch=B, max_seq=S, init="device", optimizer=torch.optim.Adam)
    opt = dm.create_optimizer(lr=1e-4)
    runs = {k: tuple(t.cuda() if t is not None else None for t in v) for k, v in batches(cfg).items()}

    def step(ids, mask, labels):
        opt.zero_grad()
        out = dm(ids, attention_mask=mask, labels=labels) if mask is not None else dm(ids, labels=labels)
        out.loss.backward()
        opt.step()

    for v in runs.values():                     # warm-up: tensor maps, first-use attributes, allocator
        for _ in range(2):
            step(*v)
    times = {k: [] for k in runs}
    for _ in range(rounds):
        for k, v in runs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                step(*v)
            opt.wait()
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) / steps)
    res = {}
    for k, ts in times.items():
        m = statistics.median(ts)
        real = B * S if k == "dense" else sum(LENGTHS)
        res[f"{k}_step_ms"] = round(m * 1e3, 2)
        res[f"{k}_samples_s"] = round(B / m, 1)
        res[f"{k}_real_tok_s"] = round(real / m, 0)
    del dm, opt
    torch.cuda.empty_cache()
    return cfg, res


def bench_attn_bwd(cfg, iters=50):
    """tl_attn_bwd_rows vs tl_attn_bwd at [8, 512] with the left padding above (CUDA events, mean over iters)."""
    from tensorlink_b200 import native as nat
    B, n_h, n_kv, d = len(LENGTHS), cfg.n_heads, cfg.n_kv_heads, cfg.head_dim
    g = torch.Generator(device="cuda").manual_seed(0)
    q = (torch.randn(B, S, n_h, d, device="cuda", generator=g) * 0.7).bfloat16()
    kc = (torch.randn(B, n_kv, S, d, device="cuda", generator=g) * 0.7).bfloat16()
    vc = torch.randn(B, n_kv, S, d, device="cuda", generator=g).bfloat16()
    do = torch.randn(B, S, n_h * d, device="cuda", generator=g).bfloat16()
    starts = torch.tensor([S - L for L in LENGTHS], dtype=torch.int32, device="cuda")
    out = torch.empty(B, S, n_h * d, dtype=torch.bfloat16, device="cuda")
    lse = torch.empty(B, n_h, S, dtype=torch.float32, device="cuda")
    dq = torch.empty_like(q)
    dk = torch.empty(B, n_h, S, d, dtype=torch.bfloat16, device="cuda")
    dv = torch.empty_like(dk)
    ws = torch.empty(nat.attn_bwd_ws(B, S, n_h), dtype=torch.uint8, device="cuda")
    scale = d ** -0.5
    res = {}
    for k, ks in (("plain", None), ("rows", starts)):
        nat.attn_prefill_fwd(q, kc, vc, out, lse, B, S, 0, n_h, n_kv, d, scale, kv_start=ks)
        for _ in range(5):
            nat.attn_bwd(q, kc, vc, out, do, lse, dq, dk, dv, ws, B, S, n_h, n_kv, d, scale, kv_start=ks)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            nat.attn_bwd(q, kc, vc, out, do, lse, dq, dk, dv, ws, B, S, n_h, n_kv, d, scale, kv_start=ks)
        e1.record()
        torch.cuda.synchronize()
        res[f"attn_bwd_{k}_us"] = round(e0.elapsed_time(e1) * 1e3 / iters, 1)
    res["attn_bwd_rows_over_plain"] = round(res["attn_bwd_rows_us"] / res["attn_bwd_plain_us"], 3)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="Qwen/Qwen2.5-0.5B")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    cfg, res = bench_step(a.model, a.rounds, a.steps)
    res.update(bench_attn_bwd(cfg))
    res = {"model": a.model, "device": torch.cuda.get_device_name(0), "power_limit_w": _power_limit(), "batch": len(LENGTHS),
           "seq": S, "lengths": list(LENGTHS), "rounds": a.rounds, "steps_per_round": a.steps, **res}
    print(json.dumps(res), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(res) + "\n")


if __name__ == "__main__":
    main()
