"""Runs the decode chain's GEMV jobs in a fresh process, in one of two modes.

    python tests/chain_env_worker.py OUT.json
        a GEMV-job set and a full-layer chain under the settings the library reads once (TL_CHAIN_STAGE_KB,
        TL_CHAIN_DYNAMIC, TL_CHAIN_L2_AHEAD_KB, TL_PDL); writes {"errors": [...], "bits": {case/leg or layer/M: sha-256
        of the outputs}, "geometry": {M/K: [slot bytes, slots, NW, K chunk]}, "dirty": [...]}.  A pair is always
        computed by one warp in ascending K with the same K chunking, so every setting must give the default's bits.

    python tests/chain_env_worker.py OUT.json --gemv-paths
        every group of tests/test_decode_chain_jobs_gpu.py's GEMV-job cases as one-job chains (both legs, guards), then
        tl_gemv_bf16 on the same inputs inside one torch.profiler session, which proves the kernel each call ran; writes
        {group: {"errors", "bits", "bound", "ratio", "path_error", "dirty"}}.  Only this process turns on CUPTI
        activity tracing, and every chain kernel here has finished before it does: the pytest process that runs the
        chain kernels, graph captures and models of that file never profiles."""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from tests import chain_cases as CC  # noqa: E402
from tests import linear_cases as L  # noqa: E402

# TL_CHAIN_STAGE_KB values and the consumer warp count each gives on the 0.5B layer at M = 1 (tests/test_chain_cases_cpu.py)
STAGE_KB = {"nw8": 8, "nw7": 9, "nw6": 30, "nw5": 36, "nw4": 44}


def _bits(ts):
    h = hashlib.sha256()
    for t in ts:
        h.update(t.contiguous().view(torch.int16).cpu().numpy().tobytes())
    return h.hexdigest()


def main(out_path):
    from tensorlink_b200 import native as nat
    from tensorlink_b200.ml import configs as C
    nat.require_device()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    kb = int(os.environ.get("TL_CHAIN_STAGE_KB", "0") or 0)
    res = {"errors": [], "bits": {}, "geometry": {}, "dirty": []}
    launch = CC.chain_gemv_launch(nat)
    cases = CC.model_gemv_jobs(C.QWEN25_05B, (1, 2)) + CC.model_gemv_jobs(C.TINY_QWEN3, (1, 2)) + CC.edge_gemv_jobs((1, 2))
    for c in cases:
        if CC.ring_geometry(c.M, c.K, kb) is None:
            continue
        for leg in ("exact", "round"):
            if leg == "exact" and not c.exact_ok:
                continue
            r = L.check_call(c, leg, launch, "cuda", sms, want_bits=True)
            res["errors"] += r["errors"]
            res["bits"][f"{c.name}/{leg}"] = r["bits_c"]
    res["dirty"] += launch.dirty
    cfg, T_max, pos = C.QWEN25_05B, 512, 300
    cos, sin = CC.rope_tables(nat, cfg, T_max)
    for M in (1, 2):
        res["geometry"][f"{M}/{cfg.intermediate}"] = list(nat.decode_chain_geometry(M, cfg.intermediate) or [])
        lay, nxt = CC.ChainLayer(cfg, M, pos, T_max, 5), CC.ChainLayer(cfg, M, 0, T_max, 6)
        b = CC.ChainBufs(cfg, M)
        g = torch.Generator(device="cuda").manual_seed(7)
        b.x.copy_(torch.randn(M, cfg.hidden, generator=g, device="cuda"))
        b.qkv.copy_(torch.randn(M, cfg.qkv_dim, generator=g, device="cuda"))
        sync = torch.zeros(nat.CHAIN_SYNC_BYTES // 4, dtype=torch.int32, device="cuda")
        ws = torch.empty(nat.decode_chain_ws(M, cfg.n_heads, cfg.n_kv_heads, cfg.head_dim), dtype=torch.uint8, device="cuda")
        posd = torch.tensor([pos], dtype=torch.int32, device="cuda")
        nat.DecodeChain(CC.layer_jobs(nat, cfg, lay, nxt, b, posd, cos, sin, T_max), M, sync, ws).launch()
        torch.cuda.synchronize()
        if sync.any():
            res["dirty"].append((f"layer/{M}", sync.nonzero()[:8, 0].tolist()))
        res["bits"][f"layer/{M}"] = _bits(b.state() + [lay.kc[:, :, pos], lay.vc[:, :, pos]])
    with open(out_path, "w") as f:
        json.dump(res, f)


def gemv_groups():
    """group name -> GEMV-job cases of tests/test_decode_chain_jobs_gpu.py"""
    from tensorlink_b200.ml import configs as C
    groups = {cfg.name: CC.model_gemv_jobs(cfg) for cfg in
              (C.QWEN25_05B, C.QWEN25_7B, C.QWEN3_8B, C.TINY_QWEN2, C.TINY_QWEN2_D128, C.TINY_QWEN3)}
    groups.update({f"edges.m{M}": CC.edge_gemv_jobs((M,)) for M in (1, 2, 3, 4)})
    return groups


def stream_path(c, sms):
    """tl_gemv_bf16 runs gemv_stream_kernel for every row chunk of this case (tests/linear_cases.py's dispatch model)"""
    return all(k.startswith("gemv_stream_kernel") for k, _ in L.gemv_path(c, sms, {})["kernels"])


def gemv_paths(out_path):
    from tensorlink_b200 import native as nat
    nat.require_device()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    chain, ref = CC.chain_gemv_launch(nat), L.native_launch(nat)
    legs = lambda c: ("exact", "round") if c.exact_ok else ("round",)
    res, chain_bits = {}, {}
    for g, cases in gemv_groups().items():
        r = res[g] = {"errors": [], "bits": [], "bound": [], "refused": [], "ratio": 0.0, "path_error": ""}
        for c in cases:
            if CC.ring_geometry(c.M, c.K) is None:      # the launcher must refuse it, before writing anything
                try:
                    chain(c, L.make_buffers(c, "round", "cuda"))
                    r["errors"].append(f"{c.name}: launched although no ring fits beside its x")
                except nat.NativeError as e:
                    if "ring slots" not in str(e):
                        r["errors"].append(f"{c.name}: refused for another reason: {e}")
                r["refused"].append(c.name)
                continue
            for leg in legs(c):
                q = L.check_call(c, leg, chain, "cuda", sms, env={}, want_bits=True)
                r["errors"] += q["errors"]
                chain_bits[(c.name, leg)] = q["bits_c"]
                if leg == "round":
                    r["ratio"] = max(r["ratio"], q["ratio"])
        r["dirty"] = list(chain.dirty)
        chain.dirty.clear()
    torch.cuda.synchronize()
    expected = []
    with L.KernelLog() as log:
        for g, cases in gemv_groups().items():
            r = res[g]
            for c in cases:
                if c.name in r["refused"]:
                    continue
                if not stream_path(c, sms):
                    r["bound"].append(c.name)
                    continue
                r["bits"].append(c.name)
                for leg in legs(c):
                    q = L.check_call(c, leg, ref, "cuda", sms, env={}, want_bits=True)
                    r["errors"] += q["errors"]
                    expected.append((f"{c.name}/{leg}", q["path"]["kernels"]))
                    if q["bits_c"] != chain_bits[(c.name, leg)]:
                        r["errors"].append(f"{c.name}/{leg}: chain output differs from gemv_stream_kernel's")
    path_error = L.match_paths(expected, log.kernels, log.all_names)
    for r in res.values():
        r["path_error"] = path_error
    with open(out_path, "w") as f:
        json.dump(res, f)


if __name__ == "__main__":
    if "--gemv-paths" in sys.argv[2:]:
        gemv_paths(sys.argv[1])
    else:
        main(sys.argv[1])
