"""Left-padded batched generation: one run of the whole batch against the grouped path (one run per real length) and
a uniform batch at the longest length.  B = 8 rows with eight distinct real lengths from 32 to 256, 128 new tokens,
greedy, one GPU; the three runs alternate, and each reports new tokens per second (median over the rounds).

    python tools/bench_padded_generate.py [--models Qwen/Qwen2.5-0.5B Qwen/Qwen2.5-7B] [--rounds 3] [--out FILE]

Weights are synthetic (seeded): the timing does not depend on their values.  Prints one JSON line per model.
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

LENGTHS = (32, 61, 90, 119, 148, 177, 206, 256)
NEW = 128


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def _timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def bench(name, rounds):
    from tensorlink_b200.ml import DistributedModel
    from tensorlink_b200.ml import configs as C
    from tensorlink_b200.ml import module as M
    cfg = C.get_config(name)
    B, S = len(LENGTHS), max(LENGTHS)
    dm = DistributedModel(cfg, training=False, max_batch=B, max_seq=S + NEW, init="device")
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(0, cfg.vocab, (B, S), generator=g)
    mask = torch.zeros(B, S, dtype=torch.int64)
    for b, L in enumerate(LENGTHS):
        mask[b, S - L:] = 1
    req = M._Request(NEW, (B, S), groups=M._left_pad_groups(mask))
    runs = {
        "one_run": lambda: dm.generate(ids, attention_mask=mask, max_new_tokens=NEW),
        "grouped": lambda: dm._generate_left_padded(ids, req),
        "uniform": lambda: dm.generate(ids, max_new_tokens=NEW),
    }
    for fn in runs.values():                      # warm-up: graph capture, tensor maps, first-use attributes
        fn()
    times = {k: [] for k in runs}
    for _ in range(rounds):
        for k, fn in runs.items():
            out, dt = _timed(fn)
            assert out.shape == (B, S + NEW), (k, out.shape)
            times[k].append(dt)
    res = {"model": name, "device": torch.cuda.get_device_name(0), "power_limit_w": _power_limit(), "batch": B,
           "lengths": list(LENGTHS), "new_tokens": NEW, "rounds": rounds}
    for k, ts in times.items():
        res[f"{k}_tok_s"] = round(B * NEW / statistics.median(ts), 1)
        res[f"{k}_s"] = [round(t, 4) for t in ts]
    res["one_run_over_grouped"] = round(res["one_run_tok_s"] / res["grouped_tok_s"], 2)
    del dm
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", nargs="+", default=["Qwen/Qwen2.5-0.5B", "Qwen/Qwen2.5-7B"])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lines = []
    for m in a.models:
        r = bench(m, a.rounds)
        print(json.dumps(r), flush=True)
        lines.append(r)
    if a.out:
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
