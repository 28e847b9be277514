"""The cost of generate's score log (return_dict_in_generate=True with output_scores / output_logits) on one GPU,
synthetic device-initialised weights.

Per workload, three variants alternating within each round: logging off (the plain call), scores on, scores + logits
on.  Decode ms per token is (t(NEW) - t(1)) / (NEW - 1) from host clocks around whole generate calls that end in a
device synchronise, so the end-of-call copy-out of the log (a device copy of [n, B, V] fp32 per kind and a broadcast,
a no-op on one stage) is not in it; the copy-out is timed separately with CUDA events.
Workloads: Qwen2.5-7B at B = 1, greedy and sampled (temperature 0.8, top_k 50, top_p 0.9); Qwen2.5-0.5B at B = 32,
greedy.

    python tools/bench_scores.py [--rounds 5] [--out FILE]

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

PROMPT, NEW = 32, 128
SAMPLE = dict(do_sample=True, temperature=0.8, top_k=50, top_p=0.9, seed=1)
VARIANTS = {"off": {}, "scores": dict(return_dict_in_generate=True, output_scores=True),
            "scores+logits": dict(return_dict_in_generate=True, output_scores=True, output_logits=True)}
WORKLOADS = (("Qwen/Qwen2.5-7B", 1, "greedy"), ("Qwen/Qwen2.5-7B", 1, "sampled"), ("Qwen/Qwen2.5-0.5B", 32, "greedy"))


def _timed(dm, ids, n, kw):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    dm.generate(ids, max_new_tokens=n, **kw)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def workload(dm, B, mode, rounds):
    from tensorlink_b200.ml.weights import synthetic_tokens
    ids = synthetic_tokens(dm.cfg, B, PROMPT)
    base = SAMPLE if mode == "sampled" else {}
    ref = None
    for name, kw in VARIANTS.items():                  # warm-up: every variant captures its graphs; tokens must agree
        out = dm.generate(ids, max_new_tokens=NEW, **base, **kw)
        seq = out if isinstance(out, torch.Tensor) else out.sequences
        ref = seq if ref is None else ref
        assert torch.equal(seq, ref), name
        dm.generate(ids, max_new_tokens=1, **base, **kw)
    t = {(v, n): [] for v in VARIANTS for n in (1, NEW)}
    for _ in range(rounds):
        for v, kw in VARIANTS.items():
            for n in (1, NEW):
                t[(v, n)].append(_timed(dm, ids, n, dict(base, **kw)))
    res = {}
    for v in VARIANTS:
        ms = (statistics.median(t[(v, NEW)]) - statistics.median(t[(v, 1)])) / (NEW - 1) * 1e3
        res[v] = {"decode_ms_per_token": round(ms, 4), "call_s": round(statistics.median(t[(v, NEW)]), 4)}
    off = res["off"]["decode_ms_per_token"]
    for v in ("scores", "scores+logits"):
        res[v]["vs_off"] = round(res[v]["decode_ms_per_token"] / off - 1, 4)
    # the copy-out at the end of a call: one kind, NEW columns
    st = dm.stage
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    cp = []
    for _ in range(max(rounds, 3)):
        ev[0].record()
        st.score_log_copy("scores", B, NEW)
        ev[1].record()
        torch.cuda.synchronize()
        cp.append(ev[0].elapsed_time(ev[1]))
    res["copy_out_ms_per_kind"] = round(statistics.median(cp), 4)
    res["log_bytes_per_step_per_kind"] = B * dm.cfg.vocab * 4
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from tensorlink_b200.ml import DistributedModel
    from tensorlink_b200.ml import configs as C
    torch.cuda.set_device(0)
    result = {"card": _card(), "prompt": PROMPT, "new": NEW, "rounds": a.rounds, "workloads": {}}
    dm, key = None, None
    for name, B, mode in WORKLOADS:
        if key != (name, B):
            dm = key = None
            torch.cuda.empty_cache()
            dm = DistributedModel(C.get_config(name), training=False, max_batch=B, max_seq=PROMPT + NEW + 16, init="device")
            key = (name, B)
        result["workloads"][f"{name} B={B} {mode}"] = workload(dm, B, mode, a.rounds)
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
