"""Prompt-lookup decoding on one GPU, batch 1, captured graphs, synthetic device-initialised weights.

(a) ms per verify step at q_len = K+1 in {2, 3, 4, 8, 11, 16} against ms per plain decode step: each round times
    STEPS graph replays of every variant back to back (the variants alternate within a round), the cache restarting
    at the same prompt each time.  The cost of a step does not depend on the weights' values.  Median and range over
    the rounds.
(b) end to end: generate NEW tokens after a self-repeating prompt with and without prompt_lookup_num_tokens=K,
    alternating; new tokens per second (median over the rounds), tokens per verify step and the first generated
    position where the two outputs differ, if they do (with synthetic weights many top-2 margins are below bf16
    resolution, so the two greedy runs may fork there).

With ``--sampled`` every variant samples at HF's defaults (temperature 1, top_k 50, SAMPLING): the decode step draws
its token and the verify step draws one token per row; the end-to-end runs use one fixed seed.

    python tools/bench_prompt_lookup.py [--model Qwen/Qwen2.5-7B] [--rounds 5] [--sampled] [--out FILE]

Prints one JSON line, with the card's name, power limit and max SM clock read in the same run.
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

Q_LENS = (2, 3, 4, 8, 11, 16)
STEPS = 32
PROMPT = 128
SAMPLING = {"temperature": 1.0, "top_k": 50, "top_p": 1.0, "seed": 1234}


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                              "-i", "0"], capture_output=True, text=True, timeout=10).stdout.strip().splitlines()[0]
        name, pl, clk = (s.strip() for s in out.split(","))
        return {"device": name, "power_limit_w": float(pl), "max_sm_clock_mhz": int(float(clk))}
    except Exception:
        return {"device": torch.cuda.get_device_name(0), "power_limit_w": None, "max_sm_clock_mhz": None}


def _spread(ts):
    return {"median": round(statistics.median(ts), 4), "min": round(min(ts), 4), "max": round(max(ts), 4)}


def step_costs(model, rounds, sampled=False):
    """(a): ms per graph replay of the plain decode step and of the verify step at each q_len."""
    from tensorlink_b200.ml import DistributedModel
    from tensorlink_b200.ml.weights import synthetic_tokens
    dm = DistributedModel(model, training=False, max_batch=1, max_seq=PROMPT + STEPS * 16 + 64, init="device")
    st, cfg = dm.stage, dm.cfg
    grp = st.slots[0]
    ids = synthetic_tokens(cfg, 1, PROMPT).cuda()
    st.set_sampling(SAMPLING if sampled else None)
    st.set_logits_processors(None)
    x = st.prefill(st.embed(ids), 0, 0)
    first = st.ids_dec[0][:1]
    st.head_argmax(x[:, -1, :].contiguous(), first, 0)
    seq = torch.cat([ids, first.view(1, 1)], dim=1)
    first_id = first.clone()

    def restart(q_len):
        """the cache back at the prompt (its keys are still there), the first token pending"""
        grp.pos_dev.fill_(PROMPT)
        grp.kvlen_dev.fill_(PROMPT)
        st.ids_dec[0][:1].copy_(first_id)
        if q_len > 1:
            st.prompt_lookup_begin(seq, q_len - 1, 2, PROMPT + STEPS * 16 + 32, [])

    def run(q_len):
        if q_len == 1:
            st.decode(0, 1, True)
        else:
            st.prompt_lookup_step(True)

    variants = (1,) + Q_LENS
    for q in variants:                                # warm-up: capture every graph
        restart(q)
        for _ in range(3):
            run(q)
    torch.cuda.synchronize()
    ms = {q: [] for q in variants}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(rounds):
        for q in variants:
            restart(q)
            torch.cuda.synchronize()
            ev[0].record()
            for _ in range(STEPS):
                run(q)
            ev[1].record()
            torch.cuda.synchronize()
            ms[q].append(ev[0].elapsed_time(ev[1]) / STEPS)
    res = {"decode_ms": _spread(ms[1])}
    for q in Q_LENS:
        res[f"verify_q{q}_ms"] = _spread(ms[q])
        res[f"verify_q{q}_over_decode"] = round(statistics.median(ms[q]) / statistics.median(ms[1]), 3)
    del dm, st, grp
    torch.cuda.empty_cache()
    return res


def end_to_end(model, rounds, K, new, period=32, times=4, sampled=False):
    """(b): tokens per second with and without prompt_lookup_num_tokens=K after a self-repeating prompt."""
    from tensorlink_b200.ml import DistributedModel
    from tensorlink_b200.ml.weights import synthetic_tokens
    cfg_prompt = period * times
    dm = DistributedModel(model, training=False, max_batch=1, max_seq=cfg_prompt + new + K + 8, init="device")
    ids = synthetic_tokens(dm.cfg, 1, period).repeat(1, times)
    kw = dict(do_sample=True, **SAMPLING) if sampled else {}
    runs = {"plain": lambda: dm.generate(ids, max_new_tokens=new, **kw),
            "lookup": lambda: dm.generate(ids, max_new_tokens=new, prompt_lookup_num_tokens=K, **kw)}
    outs = {k: fn().cpu() for k, fn in runs.items()}    # warm-up (graph capture) and the outputs compared below
    times_s = {k: [] for k in runs}
    steps = None
    for _ in range(rounds):
        for k, fn in runs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn()
            torch.cuda.synchronize()
            times_s[k].append(time.perf_counter() - t0)
            assert torch.equal(out.cpu(), outs[k]), f"{k}: not deterministic"
            if k == "lookup":
                steps = dm.timers["prompt_lookup_steps"]
    diff = (outs["plain"] != outs["lookup"])[0, cfg_prompt:].nonzero()
    res = {"prompt": cfg_prompt, "new_tokens": new, "K": K, "verify_steps": steps,
           "tokens_per_verify_step": round((new - 1) / max(steps, 1), 2),
           "first_divergence": int(diff[0]) if diff.numel() else None}
    for k, ts in times_s.items():
        res[f"{k}_tok_s"] = round(new / statistics.median(ts), 1)
        res[f"{k}_s"] = [round(t, 4) for t in ts]
    res["lookup_over_plain"] = round(res["lookup_tok_s"] / res["plain_tok_s"], 3)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="Qwen/Qwen2.5-7B")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--new", type=int, default=256)
    ap.add_argument("--sampled", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"model": a.model, **_card(), "batch": 1, "prompt_a": PROMPT, "steps_per_round": STEPS, "rounds": a.rounds,
           "sampling": SAMPLING if a.sampled else None}
    res["step_cost"] = step_costs(a.model, a.rounds, a.sampled)
    res["end_to_end"] = end_to_end(a.model, a.rounds, a.k, a.new, sampled=a.sampled)
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
