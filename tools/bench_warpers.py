"""Cost of the min_p / typical_p / epsilon_cutoff / eta_cutoff warpers on the sampled decode loop: decode ms per token
sampling without them, with each alone, with the full chain, and with the full chain and repetition_penalty, the runs
alternated within each round in one process.  Qwen2.5-7B at B = 1 and Qwen2.5-0.5B at B = 32, prompt 32 + 128 new
tokens, one GPU, captured decode graphs.  Then tl_sample and tl_sample_proc alone at V = 152,064 (CUDA events over
200 launches, alternated per round), off and with each setting.

    python tools/bench_warpers.py [--rounds 5] [--out FILE]

Weights are synthetic (seeded): the timing does not depend on their values.  The decode time is the span of the decode
rounds (CUDA events, ``generate(profile=True)``) over the 127 steps after the first token.  Prints one JSON line per
case: the median and the range (max - min) over the rounds, with the card's name and power limit.
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from tools.bench_logits_processors import _power_limit  # noqa: E402

CASES = (("Qwen/Qwen2.5-7B", 1), ("Qwen/Qwen2.5-0.5B", 32))
PROMPT, NEW = 32, 128
SAMPLE = dict(do_sample=True, temperature=0.8, top_k=50, top_p=0.9, seed=7)
CHAIN = dict(min_p=0.05, typical_p=0.9, epsilon_cutoff=3e-4, eta_cutoff=1e-3)
RUNS = {"off": {}, "min_p": dict(min_p=0.05), "typical_p": dict(typical_p=0.9), "epsilon": dict(epsilon_cutoff=3e-4),
        "eta": dict(eta_cutoff=1e-3), "chain": CHAIN, "chain_penalty": dict(CHAIN, repetition_penalty=1.2)}
KERNEL_RUNS = {"off": {}, "min_p": dict(min_p=0.05), "typical_p": dict(typical_p=0.9), "epsilon": dict(epsilon=3e-4),
               "eta": dict(eta=1e-3), "chain": dict(min_p=0.05, typical_p=0.9, epsilon=3e-4, eta=1e-3)}


def _card():
    return {"device": torch.cuda.get_device_name(0), "power_limit_w": _power_limit()}


def _summary(ms: dict) -> dict:
    out = {}
    for k, v in ms.items():
        out[f"{k}_ms"] = round(statistics.median(v), 4)
        out[f"{k}_range_ms"] = round(max(v) - min(v), 4)
    return out


def bench_decode(name, B, rounds):
    from tensorlink_b200.ml import DistributedModel
    from tensorlink_b200.ml import configs as C
    cfg = C.get_config(name)
    dm = DistributedModel(cfg, training=False, max_batch=B, max_seq=PROMPT + NEW + 8, init="device")
    ids = torch.randint(0, cfg.vocab, (B, PROMPT), generator=torch.Generator().manual_seed(0))

    def run(kw):
        out = dm.generate(ids, max_new_tokens=NEW, profile=True, **SAMPLE, **kw)
        assert out.shape == (B, PROMPT + NEW)
        return dm.timers["decode_span_s"] / (NEW - 1) * 1e3

    for kw in RUNS.values():                      # warm-up: graph capture, first-use attributes
        run(kw)
    ms = {k: [] for k in RUNS}
    for _ in range(rounds):
        for k, kw in RUNS.items():
            ms[k].append(run(kw))
    res = {"what": "decode_ms_per_token", "model": name, "batch": B, "prompt": PROMPT, "new_tokens": NEW, **_card(),
           "rounds": rounds, "sampling": SAMPLE, "chain": CHAIN, **_summary(ms)}
    del dm
    torch.cuda.empty_cache()
    return res


def bench_kernels(rounds, M=1, V=152_064, n=200):
    from tensorlink_b200 import native as nat
    g = torch.Generator().manual_seed(1)
    lg = (torch.randn(M, V, generator=g) * 2.5).to(torch.bfloat16).cuda()
    ids = torch.empty(M, dtype=torch.int64, device="cuda")
    ctr = torch.zeros(M, dtype=torch.int32, device="cuda")
    ws = torch.empty(nat.sample_ws(M), dtype=torch.uint8, device="cuda")
    L = 64
    log = torch.zeros(M, L, dtype=torch.int32, device="cuda")
    ln = torch.zeros(M, dtype=torch.int32, device="cuda")
    bt = torch.zeros(M, (V + 31) // 32, dtype=torch.int32, device="cuda")
    nat.history_fill(torch.randint(0, V, (M, 32), generator=g).cuda(), log, ln, bt, V)
    params = nat.lp_params(1.2, 0, 0, 32, []).cuda()
    pws = torch.empty(nat.logits_proc_ws(M, V), dtype=torch.uint8, device="cuda")
    s = SAMPLE

    def time_one(proc, kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            if proc:
                nat.sample_proc(lg, ids, log, ln, bt, params, ctr, pws, s["temperature"], s["top_k"], s["top_p"], 7, **kw)
            else:
                nat.sample(lg, ids, ctr, ws, s["temperature"], s["top_k"], s["top_p"], 7, **kw)
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / n * 1e3             # microseconds per launch

    out = []
    for proc in (False, True):
        for kw in KERNEL_RUNS.values():
            time_one(proc, kw)
        us = {k: [] for k in KERNEL_RUNS}
        for _ in range(rounds):
            for k, kw in KERNEL_RUNS.items():
                us[k].append(time_one(proc, kw))
        res = {"what": "kernel_us_per_launch", "kernel": "tl_sample_proc" if proc else "tl_sample", "M": M, "V": V,
               "launches": n, **_card(), "rounds": rounds,
               **{k.replace("_ms", "_us"): v for k, v in _summary(us).items()}}
        out.append(res)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--kernels-only", action="store_true")
    args = ap.parse_args()
    from tensorlink_b200 import native
    native.require_device()
    lines = []
    results = bench_kernels(args.rounds)
    if not args.kernels_only:
        results += [bench_decode(name, B, args.rounds) for name, B in CASES]
    for res in results:
        print(json.dumps(res), flush=True)
        lines.append(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
