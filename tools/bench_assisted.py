"""Assisted decoding on one GPU, batch 1, captured graphs, synthetic device-initialised weights.

(a) ms per round for K in KS with a Qwen2.5-7B model and a Qwen2.5-0.5B assistant at context PROMPT, against ms per
    plain 7B decode step.  Each round of the measurement times STEPS graph replays of every variant back to back (the
    variants alternate), the cache restarting at the same prompt each time; the assistant's part is timed the same way
    from a graph of that part alone, and the model's part is the difference.  The cost of a round does not depend on
    the weights' values.  Median and range over the rounds.  ``break_even_tokens`` = round / decode: the tokens a round
    has to emit to match plain decoding.
(b) the default K: the K with the most expected tokens per ms, E(K) / round_ms(K), where E(K) = (1 - a^(K+1)) / (1 - a)
    is the expected number of tokens a round emits when each draft agrees with the model with probability a = ALPHA,
    independently.  ALPHA is an assumption, not a measurement: no real checkpoints are at hand.
(c) the all-accept ceiling: a Qwen2.5-0.5B model with an identical assistant (every draft is accepted up to bf16 near
    ties), tokens per second against plain decoding, end to end through generate.
(d) end to end with the 7B model's first two layers (with its embedding and head) as the assistant, against plain 7B
    decoding.  The acceptance is a property of the synthetic weights, not of real checkpoints.

With ``--sampled`` every variant samples at HF's defaults (temperature 1, top_k 50, SAMPLING): the decode step draws
its token, the assistant samples its drafts and the round keeps them by speculative sampling; the end-to-end runs use
one fixed seed.  (a) then splits a round three ways: the assistant's part, the accept part (``tl_spec_accept``, both
launches, timed alone with events over ACCEPT_REPS calls on the round's own rows) and the model's part (the rest).
(e), sampled only: ``tl_spec_accept`` at K in ACCEPT_KS against one ``tl_sample`` row of the model's vocabulary.

    python tools/bench_assisted.py [--rounds 5] [--new 256] [--sampled] [--out FILE]

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

from bench_prompt_lookup import _card, _spread  # noqa: E402

KS = (1, 2, 3, 4, 5, 8, 15)
STEPS = 32
PROMPT = 128
ALPHA = 0.8
TARGET, ASSISTANT = "Qwen/Qwen2.5-7B", "Qwen/Qwen2.5-0.5B"
SAMPLING = {"temperature": 1.0, "top_k": 50, "top_p": 1.0, "seed": 1234}
ACCEPT_KS = (1, 2, 4, 8, 15)
ACCEPT_REPS = 200


def _expected_tokens(K, alpha=ALPHA):
    return (1 - alpha ** (K + 1)) / (1 - alpha)


def accept_costs(st, ast, Ks):
    """ms per tl_spec_accept call (both launches) at each K, and per one-row tl_sample call, on the rows a round left"""
    from tensorlink_b200 import native as nat
    from tensorlink_b200.ml.stage import CTR_ACCEPT
    pl, s = st.pl, SAMPLING
    warp = (s["temperature"], s["top_k"], s["top_p"], s["seed"])
    ctr = pl["ctr"][CTR_ACCEPT:CTR_ACCEPT + 1]
    ids, ws1 = torch.zeros(16, dtype=torch.int64, device=st.device), torch.empty(nat.sample_ws(1), dtype=torch.uint8,
                                                                                 device=st.device)
    calls = {f"spec_accept_k{K}": (lambda K=K: nat.spec_accept(pl["logits"][:K + 1], ast.asst["q"][:K], pl["in_ids"],
                                                               pl["n_cand"], ctr, ids, pl["spec_ws"], *warp))
             for K in Ks}
    calls["sample_1row"] = lambda: nat.sample(pl["logits"][:1], ids[:1], ctr, ws1, *warp)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ms = {}
    for name, fn in calls.items():
        for _ in range(10):
            fn()
        ev[0].record()
        for _ in range(ACCEPT_REPS):
            fn()
        ev[1].record()
        torch.cuda.synchronize()
        ms[name] = round(ev[0].elapsed_time(ev[1]) / ACCEPT_REPS, 4)
    return ms


def round_costs(rounds, sampled=False):
    """(a) and (b), and (e) when sampled"""
    from tensorlink_b200.ml import DistributedModel
    from tensorlink_b200.ml.stage import CTR_DRAFTS
    from tensorlink_b200.ml.weights import synthetic_tokens
    max_len = PROMPT + STEPS * 16 + 32
    dm = DistributedModel(TARGET, training=False, max_batch=1, max_seq=max_len + 32, init="device")
    draft = DistributedModel(ASSISTANT, training=False, max_batch=1, max_seq=max_len + 32, init="device")
    st, ast = dm.stage, draft.stage
    grp = st.slots[0]
    ids = synthetic_tokens(dm.cfg, 1, PROMPT).cuda()
    st.set_sampling(SAMPLING if sampled else None)
    st.set_logits_processors(None)
    x = st.prefill(st.embed(ids), 0, 0)
    first = st.ids_dec[0][:1]
    st.head_argmax(x[:, -1, :].contiguous(), first, 0)
    ast.prefill(ast.embed(ids), 0, 0)
    seq = torch.cat([ids, first.view(1, 1)], dim=1)
    first_id = first.clone()
    part_graphs = {}

    def restart(K):
        """the cache back at the prompt (its keys are still there), the first token pending"""
        grp.pos_dev.fill_(PROMPT)
        grp.kvlen_dev.fill_(PROMPT)
        st.ids_dec[0][:1].copy_(first_id)
        if K:
            st.prompt_lookup_begin(seq, K, 0, max_len, [], assistant=ast)

    def assistant_part(K):
        g = part_graphs.get(K)
        if g is None:
            args = (st.hist_log[0, 0], st.hist_len[0, :1], st.pl["in_ids"], K,
                    (SAMPLING, st.pl["ctr"][CTR_DRAFTS:CTR_DRAFTS + 1]) if sampled else None)
            ast.assist_draft(*args)                   # warm-up outside capture
            torch.cuda.synchronize()
            g = part_graphs[K] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                ast.assist_draft(*args)
        g.replay()

    variants = [("decode", 0)] + [(f"round_k{K}", K) for K in KS] + [(f"assistant_k{K}", K) for K in KS]

    def run(name, K):
        if name == "decode":
            st.decode(0, 1, True)
        elif name.startswith("round"):
            st.prompt_lookup_step(True)
        else:
            assistant_part(K)

    for name, K in variants:                          # warm-up: capture every graph
        restart(K)
        for _ in range(3):
            run(name, K)
    torch.cuda.synchronize()
    ms = {name: [] for name, _ in variants}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(rounds):
        for name, K in variants:
            restart(K)
            torch.cuda.synchronize()
            ev[0].record()
            for _ in range(STEPS):
                run(name, K)
            ev[1].record()
            torch.cuda.synchronize()
            ms[name].append(ev[0].elapsed_time(ev[1]) / STEPS)
    dec = statistics.median(ms["decode"])
    res = {"decode_ms": _spread(ms["decode"]), "per_k": {}}
    acc = {}
    if sampled:
        restart(max(KS))
        st.prompt_lookup_step(True)                   # a round's rows in the buffers
        acc = accept_costs(st, ast, sorted(set(KS) | set(ACCEPT_KS)))
        res["accept_ms"] = {k: v for k, v in acc.items() if k == "sample_1row" or int(k.split("_k")[1]) in ACCEPT_KS}
    best = None
    for K in KS:
        r, a = statistics.median(ms[f"round_k{K}"]), statistics.median(ms[f"assistant_k{K}"])
        rate = _expected_tokens(K) / r
        c = acc.get(f"spec_accept_k{K}", 0.0)
        res["per_k"][K] = {"round_ms": _spread(ms[f"round_k{K}"]), "assistant_ms": _spread(ms[f"assistant_k{K}"]),
                           "model_ms": round(r - a - c, 4), "break_even_tokens": round(r / dec, 3),
                           "expected_tokens_at_alpha": round(_expected_tokens(K), 3),
                           "expected_tok_per_ms": round(rate, 4), "expected_over_plain": round(rate * dec, 3)}
        if sampled:
            res["per_k"][K]["accept_ms"] = c
        if best is None or rate > best[1]:
            best = (K, rate)
    res["default_k"] = {"K": best[0], "alpha": ALPHA,
                        "rule": "argmax over K of E(K) / round_ms(K), E(K) = (1 - alpha^(K+1)) / (1 - alpha)"}
    del dm, draft, st, ast, grp, part_graphs
    torch.cuda.empty_cache()
    return res


def _e2e(dm, draft, ids, new, rounds, Ks, sampled=False):
    kw = dict(do_sample=True, **SAMPLING) if sampled else {}
    runs = {"plain": lambda: dm.generate(ids, max_new_tokens=new, **kw)}
    for K in Ks:
        runs[f"k{K}"] = (lambda K=K: dm.generate(ids, max_new_tokens=new, assistant_model=draft, num_assistant_tokens=K,
                                                 **kw))
    outs = {k: fn().cpu() for k, fn in runs.items()}    # warm-up (graph capture) and the outputs compared below
    times_s = {k: [] for k in runs}
    steps = {}
    for _ in range(rounds):
        for k, fn in runs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn()
            torch.cuda.synchronize()
            times_s[k].append(time.perf_counter() - t0)
            assert torch.equal(out.cpu(), outs[k]), f"{k}: not deterministic"
            if k != "plain":
                steps[k] = dm.timers["assisted_steps"]
    S = ids.shape[1]
    res = {"prompt": S, "new_tokens": new, "plain_tok_s": round(new / statistics.median(times_s["plain"]), 1)}
    for K in Ks:
        k = f"k{K}"
        diff = (outs["plain"] != outs[k])[0, S:].nonzero()
        tok_s = new / statistics.median(times_s[k])
        res[k] = {"tok_s": round(tok_s, 1), "over_plain": round(tok_s / res["plain_tok_s"], 3), "rounds": steps[k],
                  "tokens_per_round": round((new - 1) / max(steps[k], 1), 2),
                  "first_divergence": int(diff[0]) if diff.numel() else None,
                  "s": [round(t, 4) for t in times_s[k]]}
    res["plain_s"] = [round(t, 4) for t in times_s["plain"]]
    return res


def all_accept(rounds, new, Ks, sampled=False):
    """(c)"""
    from tensorlink_b200.ml import DistributedModel
    from tensorlink_b200.ml.weights import synthetic_tokens
    kw = dict(training=False, max_batch=1, max_seq=PROMPT + new + 32, init="device")
    dm, draft = DistributedModel(ASSISTANT, **kw), DistributedModel(ASSISTANT, **kw)
    ids = synthetic_tokens(dm.cfg, 1, PROMPT)
    res = {"model": ASSISTANT, "assistant": "the same weights", **_e2e(dm, draft, ids, new, rounds, Ks, sampled)}
    del dm, draft
    torch.cuda.empty_cache()
    return res


def truncated(rounds, new, Ks, sampled=False):
    """(d)"""
    from tensorlink_b200.ml import DistributedModel
    from tensorlink_b200.ml.configs import get_config
    from tensorlink_b200.ml.weights import synthetic_tokens
    kw = dict(training=False, max_batch=1, max_seq=PROMPT + new + 32, init="device")
    dm = DistributedModel(TARGET, **kw)
    draft = DistributedModel(get_config(TARGET).scaled(n_layers=2), **kw)
    for name, t in draft.stage.params.v.items():      # the embedding, the head, the final norm and layers 0 and 1
        t.copy_(dm.stage.params.v[name])
    ids = synthetic_tokens(dm.cfg, 1, PROMPT)
    res = {"model": TARGET, "assistant": "its first 2 of 28 layers, embedding and head (synthetic weights)",
           **_e2e(dm, draft, ids, new, rounds, Ks, sampled)}
    del dm, draft
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--new", type=int, default=256)
    ap.add_argument("--sampled", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"model": TARGET, "assistant_model": ASSISTANT, **_card(), "batch": 1, "prompt": PROMPT,
           "steps_per_round": STEPS, "rounds": a.rounds, "sampling": SAMPLING if a.sampled else None}
    res["round_cost"] = round_costs(a.rounds, a.sampled)
    Ks = sorted({1, 2, 4, 8, 15, res["round_cost"]["default_k"]["K"]})
    res["all_accept"] = all_accept(a.rounds, a.new, Ks, a.sampled)
    res["truncated_assistant"] = truncated(a.rounds, a.new, Ks, a.sampled)
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
