"""FP8 (HF fine-grained, weight-only) against bf16 on one GPU, synthetic device-initialised weights quantized on the device.

Per model (Qwen2.5-7B, Qwen3-8B), the bf16 and the FP8 model side by side, variants alternating within each round:
(a) batch-1 greedy generate, prompt PROMPT + NEW tokens: end-to-end tok/s, decode ms per token ((t(NEW) - t(1)) /
    (NEW - 1)), HBM bytes per token (algorithmic: the decoder Linears' weights, FP8 plus their fp32 scales or bf16, the
    bf16 lm_head) and that stream's share of the 3.35 TB/s data-sheet bound.
(b) the decode Linears alone (gate/up with the SwiGLU epilogue and the norm prologue, down with the residual), one row,
    timed with CUDA events over REPS launches: achieved TB/s of algorithmic bytes.
(c) prefill of PREFILLS tokens (one row, the stage's layers only).
(d) the row threshold: one captured decode step at B rows and one captured verify step of q_len rows, with the FP8
    GEMV in passes of at most 4 rows ("gemv", up to 8 rows) against dequantize-then-GEMM ("scratch"); bf16 beside them.

    python tools/bench_fp8.py [--rounds 5] [--out FILE]

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

MODELS = ("Qwen/Qwen2.5-7B", "Qwen/Qwen3-8B")
QC = {"quant_method": "fp8", "fmt": "e4m3", "activation_scheme": "dynamic", "weight_block_size": [128, 128]}
PROMPT, NEW = 32, 128
PREFILLS = (32, 512)
DECODE_B = (4, 8, 32)
VERIFY_N = (4, 6, 8, 12, 16)
REPS = 200
HBM_TBS = 3.35


def _med(xs):
    return round(statistics.median(xs), 4)


def _stream_bytes(dm):
    p = dm.stage.params
    lin = sum(t.numel() * t.element_size() for n, t in p.v.items() if n.split(".")[-1] in ("wqkv", "wo", "wgu", "wd"))
    sc = p.scales.numel() * 4 if p.fp8 else 0
    return lin + sc + p.v["head"].numel() * 2


def e2e(dms, rounds):
    """(a)"""
    from tensorlink_b200.ml.weights import synthetic_tokens
    ids = synthetic_tokens(dms["bf16"].cfg, 1, PROMPT)
    outs = {k: dm.generate(ids, max_new_tokens=NEW).cpu() for k, dm in dms.items()}      # warm-up (graph capture)
    for dm in dms.values():
        dm.generate(ids, max_new_tokens=1)
    t = {(k, n): [] for k in dms for n in (1, NEW)}
    for _ in range(rounds):
        for k, dm in dms.items():
            for n in (1, NEW):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                dm.generate(ids, max_new_tokens=n)
                torch.cuda.synchronize()
                t[(k, n)].append(time.perf_counter() - t0)
    res = {"same_tokens": bool(torch.equal(outs["bf16"], outs["fp8"]))}
    for k, dm in dms.items():
        dec = [(a - b) / (NEW - 1) for a, b in zip(t[(k, NEW)], t[(k, 1)])]
        ms = statistics.median(dec) * 1e3
        by = _stream_bytes(dm)
        res[k] = {"tok_s": round(NEW / statistics.median(t[(k, NEW)]), 1), "decode_ms_per_token": round(ms, 3),
                  "decode_ms_range": [round(min(dec) * 1e3, 3), round(max(dec) * 1e3, 3)],
                  "bytes_per_token_GB": round(by / 1e9, 3), "share_of_bound": round(by / (HBM_TBS * 1e12) / (ms * 1e-3), 3)}
    res["decode_speedup"] = round(res["bf16"]["decode_ms_per_token"] / res["fp8"]["decode_ms_per_token"], 3)
    return res


def _events(fn, reps=REPS):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def linears(dms, rounds):
    """(b)"""
    from tensorlink_b200 import native as nat
    res = {}
    for name, flags in (("wgu", nat.EPI_SWIGLU), ("wd", nat.EPI_RESIDUAL)):
        t = {k: [] for k in dms}
        for _ in range(rounds):
            for k, dm in dms.items():
                grp, p = dm.stage.slots[0], dm.stage.params
                li = p.layer_ids[0]
                w = p.v[f"l{li}.{name}"]
                N, K = w.shape
                x = torch.randn(1, K, device=w.device).to(torch.bfloat16)
                kw = {"norm_w": p.v[f"l{li}.ln2"]} if name == "wgu" else {"residual": torch.zeros(1, N, device=w.device,
                                                                                                dtype=torch.bfloat16)}
                t[k].append(_events(lambda: grp._gemv(x, f"l{li}.{name}", flags=flags if name == "wgu" else 0, **kw)))
        for k, dm in dms.items():
            p = dm.stage.params
            w = p.v[f"l{p.layer_ids[0]}.{name}"]
            by = w.numel() * w.element_size() + (w.numel() // 128 * 4 if p.fp8 else 0)
            ms = statistics.median(t[k])
            res[f"{name}_{k}"] = {"shape": list(w.shape), "ms": round(ms, 4), "TB_s": round(by / (ms * 1e-3) / 1e12, 3)}
    return res


def prefill(dms, rounds):
    """(c)"""
    res = {}
    for S in PREFILLS:
        t = {k: [] for k in dms}
        for _ in range(rounds + 1):
            for k, dm in dms.items():
                st = dm.stage
                h = st.embed(torch.randint(0, dm.cfg.vocab, (1, S), device=st.device))
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                st.prefill(h, 0, 0)
                torch.cuda.synchronize()
                t[k].append(time.perf_counter() - t0)
        res[f"S{S}"] = {k: {"ms": round(statistics.median(v[1:]) * 1e3, 3)} for k, v in t.items()}
    return res


def _graph_ms(fn, reps=50):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    return _events(g.replay, reps)


def threshold(dms):
    """(d)"""
    res = {}
    for k, dm in dms.items():
        grp = dm.stage.slots[0]
        grp.reset_cache(PROMPT)
        H = dm.cfg.hidden
        modes = {"gemv": 8, "scratch": 0} if k == "fp8" else {"default": None}
        for mode, rows in modes.items():
            if rows is not None:
                grp.gemv_rows = lambda rows=rows: rows
            for B in DECODE_B:
                if mode == "gemv" and B > 8:
                    continue
                x = torch.randn(B, H, device=grp.device).mul_(0.1).to(torch.bfloat16)
                res[f"decode_B{B}_{k}_{mode}"] = round(_graph_ms(lambda: grp.decode_step_inplace(x, advance=False)), 4)
            for n in VERIFY_N:
                if mode == "gemv" and n > 8:
                    continue
                x = torch.randn(n, H, device=grp.device).mul_(0.1).to(torch.bfloat16)
                res[f"verify_n{n}_{k}_{mode}"] = round(_graph_ms(lambda: grp.verify_step_inplace(x)), 4)
            grp.__dict__.pop("gemv_rows", None)
    return res


def run_model(name, rounds):
    from tensorlink_b200.ml import DistributedModel
    kw = dict(training=False, max_batch=max(DECODE_B), max_seq=max(PREFILLS) + NEW + 32, init="device")
    dms = {"bf16": DistributedModel(name, **kw), "fp8": DistributedModel(name, quantization_config=QC, **kw)}
    res = {"model": name, "e2e": e2e(dms, rounds), "linears": linears(dms, rounds), "prefill": prefill(dms, rounds),
           "rows": threshold(dms)}
    del dms
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--models", default=",".join(MODELS))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8 measures on a GPU; none is visible")
    res = {**_card(), "batch": 1, "prompt": PROMPT, "new_tokens": NEW, "rounds": a.rounds,
           "models": [run_model(m, a.rounds) for m in a.models.split(",")]}
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
