"""Cost of the logits processors on the decode loop: decode ms per token with processors off and on
(repetition_penalty=1.2, no_repeat_ngram_size=3), greedy and sampled, the four runs alternated in one process.
Qwen2.5-7B at B = 1 and Qwen2.5-0.5B at B = 32, prompt 32 + 128 new tokens, one GPU.

    python tools/bench_logits_processors.py [--rounds 5] [--out FILE]

Weights are synthetic (seeded): the timing does not depend on their values.  The decode time is the span of the decode
rounds (CUDA events, ``generate(profile=True)``) over the 127 steps after the first token.  Prints one JSON line per case.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

CASES = (("Qwen/Qwen2.5-7B", 1), ("Qwen/Qwen2.5-0.5B", 32))
PROMPT, NEW = 32, 128
PROCS = dict(repetition_penalty=1.2, no_repeat_ngram_size=3)
SAMPLE = dict(do_sample=True, temperature=0.8, top_k=50, top_p=0.9, seed=7)


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def bench(name, B, rounds):
    from tensorlink_b200.ml import DistributedModel
    from tensorlink_b200.ml import configs as C
    cfg = C.get_config(name)
    dm = DistributedModel(cfg, training=False, max_batch=B, max_seq=PROMPT + NEW + 8, init="device")
    ids = torch.randint(0, cfg.vocab, (B, PROMPT), generator=torch.Generator().manual_seed(0))
    runs = {"greedy_off": {}, "greedy_on": PROCS, "sampled_off": SAMPLE, "sampled_on": {**SAMPLE, **PROCS}}

    def run(kw):
        out = dm.generate(ids, max_new_tokens=NEW, profile=True, **kw)
        assert out.shape == (B, PROMPT + NEW)
        return dm.timers["decode_span_s"] / (NEW - 1) * 1e3

    for kw in runs.values():                      # warm-up: graph capture, tensor maps, first-use attributes
        run(kw)
    ms = {k: [] for k in runs}
    for _ in range(rounds):
        for k, kw in runs.items():
            ms[k].append(run(kw))
    res = {"model": name, "batch": B, "prompt": PROMPT, "new_tokens": NEW, "device": torch.cuda.get_device_name(0),
           "power_limit_w": _power_limit(), "rounds": rounds, "processors": PROCS}
    for k, v in ms.items():
        res[f"{k}_ms_per_token"] = round(statistics.median(v), 4)
        res[f"{k}_spread_ms"] = round(max(v) - min(v), 4)
    for mode in ("greedy", "sampled"):
        res[f"{mode}_overhead_pct"] = round(100 * (res[f"{mode}_on_ms_per_token"] / res[f"{mode}_off_ms_per_token"] - 1), 2)
    del dm
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from tensorlink_b200 import native
    native.require_device()
    lines = []
    for name, B in CASES:
        res = bench(name, B, args.rounds)
        print(json.dumps(res), flush=True)
        lines.append(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
