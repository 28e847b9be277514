"""Where the decode-chain kernel's edges are (csrc/decode_chain.cu), restated in Python, and a CPU model of its attention.

The GPU tests (tests/test_decode_chain_jobs_gpu.py) place their cases with this module, the way tests/linear_cases.py
places the GEMV cases with ``gemv_stream_params``:

  * ``ring_geometry``: the shared-memory ring the launcher builds from (M, K_max, TL_CHAIN_STAGE_KB): slot bytes, slots,
    consumer warps NW and the K chunk DC_KC, or None where it cannot place the shape.
  * ``gemv_units``: how one GEMV job is cut into ring units (pairs per unit P, unit count, K chunks) and split over CTAs.
  * ``attn_partition``: the key ranges of the split-KV attention job, one CTA per range, over all CTAs of the grid.
  * ``chain_attention``: the attention job's arithmetic on one (row, kv head) group: per-CTA 32-key tiles in the log2
    domain, P rounded to bf16 before P.V, fp32 state, and the last-arriving CTA's combine.  ``fault`` plants one of the
    mistakes the GPU cases are chosen to catch.

Nothing here needs a GPU: tests/test_chain_cases_cpu.py pins hand-checked values and runs the planted faults.
"""
from __future__ import annotations

from typing import List, Optional

import torch

SMEM_CAP = 227 * 1024 - 1024            # dynamic shared memory of the kernel
DC_CW = 8                               # consumer warps
DC_MAX_STAGES = 24
DC_MAX_M = 4
DC_TILE = 32                            # keys per attention tile
DC_MIN_KEYS = 128                       # keys per CTA below which the attention job needs no combine
DC_ATTN_BYTES = 8 * 128 * 4 + 2 * 128 * 4 + 8 * DC_TILE * 4 + 2 * DC_TILE * (128 * 2 + 16)
BARRIER_BYTES = 2 * DC_MAX_STAGES * 8
LOG2E = 1.4426950408889634

FAULTS = ("stale_max", "range_off_by_one", "drop_new_key", "new_key_from_cache")


# ------------------------------------------------------------------------------------------------ ring geometry
def fixed_bytes(M: int, k_max: int) -> int:
    """x staging (M rows of K_max, 128-byte rounded) + the attention job's buffers + the ring's mbarriers"""
    return ((M * k_max * 2 + 127) & ~127) + DC_ATTN_BYTES + BARRIER_BYTES


def ring_geometry(M: int, k_max: int, stage_kb: int = 0) -> Optional[dict]:
    """tl_decode_chain_geometry: {stage_bytes, n_stages, NW, kc}, or None ("does not fit").  stage_kb as
    TL_CHAIN_STAGE_KB: 0 the default (8 slots of up to 24 KB while 12 KB fit), else a forced slot size (8 KB and up;
    smaller values force 16 KB)."""
    assert 1 <= M <= DC_MAX_M
    fixed = fixed_bytes(M, k_max)
    if fixed + 4 * 8192 > SMEM_CAP:
        return None
    stage = n_stages = nw = 0
    if not stage_kb:
        kb = min(24, (SMEM_CAP - fixed) // 8 // 1024)
        if kb >= 12:
            stage, n_stages, nw = kb * 1024, 8, 8
    if not stage:
        stage = (stage_kb if stage_kb >= 8 else 16) * 1024
        max_stages = min(DC_MAX_STAGES, (SMEM_CAP - fixed) // stage)
        if max_stages < 4:
            return None
        for w in range(DC_CW, 3, -1):
            if max_stages // w * w > n_stages:
                n_stages, nw = max_stages // w * w, w
    return {"stage_bytes": stage, "n_stages": n_stages, "NW": nw, "kc": (stage // 4) & ~7}


def gemv_units(N: int, K: int, geo: dict, grid: int) -> dict:
    """dc_geom: a unit is P consecutive row pairs (one slot) or, when a pair does not fit a slot, one pair in n_chunks
    K-chunks of kc elements (one slot each).  u_ranges: each CTA's units under the static split."""
    npairs = N // 2
    chunked = K > geo["kc"] or 4 * K > geo["stage_bytes"]
    P = 1 if chunked else min(8, geo["stage_bytes"] // (4 * K))
    U = -(-npairs // P)
    KC = geo["kc"] if chunked else K
    return {"chunked": chunked, "P": P, "units": U, "n_chunks": -(-K // KC),
            "last_unit_pairs": npairs - (U - 1) * P,
            "u_ranges": [(c * U // grid, (c + 1) * U // grid) for c in range(grid)]}


def kc_edge(M: int, stage_kb: int = 0, pairs: int = 1) -> int:
    """the largest K (a multiple of 8) with 4 * K * pairs <= the slot of its own geometry: K + 8 needs a smaller P (or,
    for pairs = 1, K-chunks).  The slot depends on K through the x staging, so this is searched, not divided."""
    best = 0
    for K in range(8, 32768, 8):
        g = ring_geometry(M, K, stage_kb)
        if g is None:
            break
        if 4 * K * pairs <= g["stage_bytes"] and K <= g["kc"]:
            best = K
    return best


# ------------------------------------------------------------------------------------------------ attention partition
def attn_partition(sms: int, n_kv: int, M: int, pos: int) -> dict:
    """The attention job's split over the grid for a new token at `pos` (keys 0..pos, key pos = the new token):
    cpg CTAs per (row, kv head) group, cpg_eff of them get whole 32-key tiles of `chunk` keys each (no empty range);
    ranges[s] = [k0, k1) of CTA s of a group; owner = the CTA whose range holds pos (it appends the new key)."""
    G = n_kv * M
    assert 1 <= G <= min(sms, 60)
    cpg = sms // G
    n_keys = pos + 1
    cpg_eff = min(cpg, -(-n_keys // DC_MIN_KEYS))
    chunk = -(-(-(-n_keys // cpg_eff)) // DC_TILE) * DC_TILE
    cpg_eff = -(-n_keys // chunk)
    ranges = [(s * chunk, min(n_keys, (s + 1) * chunk)) for s in range(cpg_eff)]
    return {"cpg": cpg, "cpg_eff": cpg_eff, "chunk": chunk, "ranges": ranges, "owner": cpg_eff - 1,
            "combine": cpg_eff > 1}


def boundary_positions(sms: int, n_kv: int, M: int, max_pos: int) -> List[int]:
    """positions on both sides of the partition's edges: the first position with 2, 3 and all cpg CTAs per group, and
    the first ones where the owner's range holds a single key (the new token starts a range) after each of those"""
    out = set()
    prev = attn_partition(sms, n_kv, M, 0)
    firsts = {}
    for pos in range(1, max_pos + 1):
        p = attn_partition(sms, n_kv, M, pos)
        if p["cpg_eff"] != prev["cpg_eff"] and p["cpg_eff"] not in firsts:
            firsts[p["cpg_eff"]] = pos
        if p["ranges"][-1][1] - p["ranges"][-1][0] == 1 and p["cpg_eff"] > 1 and len(out) < 4:
            out.update((pos - 1, pos))
        prev = p
    for ce in (2, 3, attn_partition(sms, n_kv, M, max_pos)["cpg"]):
        if ce in firsts:
            out.update((firsts[ce] - 1, firsts[ce]))
    return sorted(p for p in out if 0 <= p <= max_pos)


ATTN_GEOMS = [  # n_h, n_kv, d, q/k-norm: n_rep 1, 2, 4, 7 (d 128 and 64), 8 (d 128 and 64)
    (4, 4, 64, False), (4, 2, 128, True), (32, 8, 128, True), (28, 4, 128, False), (14, 2, 64, True),
    (32, 4, 128, False), (16, 2, 64, True)]
ATTN_PATTERNS = ["flat", "sink", "rising", "falling", "wide", "spike@T-1"]
ATTN_SHORT = [0, 1, 31, 32, 127, 128]          # first tile, tile edge, DC_MIN_KEYS: direct store vs combine
ATTN_LONG = [2047, 4095, 8191]
ATTN_T_MAX = 8192


def attn_cases(sms: int) -> List[tuple]:
    """(n_h, n_kv, d, qk_norm, M, pos, pattern) of the attention-job cases: every geometry at the short positions and
    the partition's edges, every pattern at a long context, and spikes on the first and the last key of a CTA range."""
    cs = []
    for gi, (n_h, n_kv, d, qn) in enumerate(ATTN_GEOMS):
        for pi, pos in enumerate(ATTN_SHORT):
            cs.append((n_h, n_kv, d, qn, 1 + (gi + pi) % 4, pos, ATTN_PATTERNS[(gi + pi) % len(ATTN_PATTERNS)]))
        M = 1 + gi % 4
        for pi, pos in enumerate(boundary_positions(sms, n_kv, M, ATTN_T_MAX - 1)):
            cs.append((n_h, n_kv, d, qn, M, pos, ATTN_PATTERNS[(gi + pi + 2) % len(ATTN_PATTERNS)]))
    for pi, pat in enumerate(ATTN_PATTERNS):
        n_h, n_kv, d, qn = ATTN_GEOMS[(pi + 3) % len(ATTN_GEOMS)]
        cs.append((n_h, n_kv, d, qn, 1 + pi % 4, ATTN_LONG[pi % 3], pat))
    for gi, (n_h, n_kv, d, qn) in enumerate(ATTN_GEOMS[::2]):
        M = 1 + (gi + 1) % 4
        for pos in (1000, ATTN_T_MAX - 1):
            r = attn_partition(sms, n_kv, M, pos)["ranges"]
            for j in sorted({r[0][1] - 1, r[1][0], r[-1][0], r[-2][1] - 1}):
                cs.append((n_h, n_kv, d, qn, M, pos, f"spike@{j}"))
    return cs


# ------------------------------------------------------------------------------------------------ attention CPU model
def _bf(x):
    return x.float().bfloat16().float()


def chain_attention(q, k_cache, v_cache, k_new, v_new, pos: int, scale: float, partition: dict,
                    fault: Optional[str] = None) -> torch.Tensor:
    """One (row, kv head) group of the attention job.  q [n_rep, d] (rotated), k_cache / v_cache [T, d] (rows >= pos
    are not read: the kernel takes key pos from k_new / v_new, the new token's rotated key and value), all on the bf16
    grid.  Returns out [n_rep, d] rounded to bf16.

    Faults: stale_max (the combine keeps the first partial's max and never rescales), range_off_by_one (every range
    but the last ends one key early: the boundary key belongs to no CTA), drop_new_key (key pos is left out),
    new_key_from_cache (key pos is read from the cache, which holds whatever was there before the append)."""
    q = q.float()
    ranges = list(partition["ranges"])
    if fault == "range_off_by_one":
        ranges = [(a, b - 1) if i + 1 < len(ranges) else (a, b) for i, (a, b) in enumerate(ranges)]
    keys = k_cache[:pos + 1].float().clone()
    vals = v_cache[:pos + 1].float().clone()
    if fault != "new_key_from_cache":
        keys[pos], vals[pos] = k_new.float(), v_new.float()
    parts = []
    for k0, k1 in ranges:
        m = torch.full((q.shape[0],), float("-inf"))
        l = torch.zeros(q.shape[0])
        o = torch.zeros(q.shape[0], q.shape[1])
        for t0 in range(k0, k1, DC_TILE):
            t1 = min(k1, t0 + DC_TILE)
            idx = torch.arange(t0, t1)
            if fault == "drop_new_key":
                idx = idx[idx != pos]
            if idx.numel() == 0:
                continue
            s = (q @ keys[idx].t()) * (scale * LOG2E)
            m_new = torch.maximum(m, s.amax(-1))
            p = torch.exp2(s - m_new[:, None])
            alpha = torch.exp2(m - m_new)
            l = l * alpha + p.sum(-1)
            o = o * alpha[:, None] + _bf(p) @ vals[idx]
            m = m_new
        parts.append((m, l, o))
    if len(parts) == 1:
        m, l, o = parts[0]
        return _bf(o / l[:, None])
    mc = torch.full_like(parts[0][0], float("-inf"))
    L = torch.zeros_like(parts[0][1])
    O = torch.zeros_like(parts[0][2])
    for i, (m, l, o) in enumerate(parts):
        mn = torch.maximum(mc, m)
        if fault == "stale_max" and i > 0:
            mn = mc
        a, w = torch.exp2(mc - mn), torch.exp2(m - mn)
        L = L * a + w * l
        O = O * a[:, None] + w[:, None] * o
        mc = mn
    return _bf(O / L[:, None])


# ------------------------------------------------------------------------------------------------ launches (GPU side)
def chain_gemv_launch(nat):
    """launch(c, bufs) for linear_cases.check_call: the GEMV case as a one-job chain (x, W, y, residual contiguous with
    pitch = row length, inside their guards).  Every launch is followed by a check that the sync slot is back to
    zero; the words that are not are appended to ``launch.dirty``."""
    from tests import linear_cases as L
    state = {}

    def ptr(bufs, k):
        return bufs[k].ptr if k in bufs else None

    def launch(c, bufs):
        dev = bufs["a"].buf.device
        if not state:
            state["sync"] = torch.zeros(nat.CHAIN_SYNC_BYTES // 4, dtype=torch.int32, device=dev)
            state["ws"] = torch.empty(256, dtype=torch.uint8, device=dev)
        C = bufs["c"]
        job = nat.make_job(nat.JOB_GEMV, N=c.N, K=c.K, flags=c.flags, W=bufs["b"].ptr, x=bufs["a"].ptr, y=C.ptr,
                           bias=ptr(bufs, "bias"), residual=C.ptr if c.alias else ptr(bufs, "res"),
                           norm_w=ptr(bufs, "g"), eps=L.EPS)
        nat.DecodeChain([job], c.M, state["sync"], state["ws"]).launch()
        nz = state["sync"].nonzero()
        if nz.numel():
            launch.dirty.append((c.name, nz[:8, 0].tolist()))
            state["sync"].zero_()

    launch.dirty = []
    return launch


class ChainLayer:
    """Random weights of one decoder layer of `cfg` (std 0.02, norm gains 1 + 0.1 N(0,1)) and its KV caches for M rows
    (keys and values of positions < pos random, NaN above)."""

    def __init__(self, cfg, M, pos, T_max, seed, device="cuda"):
        g = torch.Generator(device=device).manual_seed(seed)
        bf = torch.bfloat16

        def rn(*shape, std=0.02, mean=0.0):
            return (torch.randn(*shape, generator=g, device=device) * std + mean).to(bf)

        H, I, Q, QKV, d = cfg.hidden, cfg.intermediate, cfg.q_dim, cfg.qkv_dim, cfg.head_dim
        self.wqkv, self.wo, self.wgu, self.wd = rn(QKV, H), rn(H, Q), rn(2 * I, H), rn(H, I)
        self.bqkv = rn(QKV, std=0.1) if cfg.qkv_bias else None
        self.ln1, self.ln2 = rn(H, std=0.1, mean=1.0), rn(H, std=0.1, mean=1.0)
        self.qn = rn(d, std=0.1, mean=1.0) if cfg.qk_norm else None
        self.kn = rn(d, std=0.1, mean=1.0) if cfg.qk_norm else None
        self.kc = torch.full((M, cfg.n_kv_heads, T_max, d), float("nan"), dtype=bf, device=device)
        self.vc = torch.full_like(self.kc, float("nan"))
        if pos:
            self.kc[:, :, :pos] = rn(M, cfg.n_kv_heads, pos, d, std=1.0)
            self.vc[:, :, :pos] = rn(M, cfg.n_kv_heads, pos, d, std=1.0)


class ChainBufs:
    def __init__(self, cfg, M, device="cuda"):
        bf = torch.bfloat16
        self.x = torch.empty(M, cfg.hidden, dtype=bf, device=device)
        self.qkv = torch.empty(M, cfg.qkv_dim, dtype=bf, device=device)
        self.attn = torch.empty(M, cfg.q_dim, dtype=bf, device=device)
        self.act = torch.empty(M, cfg.intermediate, dtype=bf, device=device)

    def state(self):
        return [t.clone() for t in (self.x, self.qkv, self.attn, self.act)]


def layer_jobs(nat, cfg, layer: ChainLayer, nxt: ChainLayer, b: ChainBufs, pos_dev, cos, sin, T_max, flags=0):
    """[ATTN, o, gate/up, down, qkv of the next layer] as ml/shard.py builds a layer's chain"""
    J = nat.make_job
    return [J(nat.JOB_ATTN, x=b.qkv, y=b.attn, k_cache=layer.kc, v_cache=layer.vc, pos_dev=pos_dev, cos_tab=cos, sin_tab=sin,
              q_norm_w=layer.qn, k_norm_w=layer.kn, n_h=cfg.n_heads, n_kv=cfg.n_kv_heads, d=cfg.head_dim, T_max=T_max,
              scale=cfg.head_dim ** -0.5, eps=cfg.rms_eps, flags=flags),
            J(nat.JOB_GEMV, N=cfg.hidden, K=cfg.q_dim, flags=nat.EPI_RESIDUAL, W=layer.wo, x=b.attn, y=b.x, residual=b.x),
            J(nat.JOB_GEMV, N=2 * cfg.intermediate, K=cfg.hidden, flags=nat.EPI_SWIGLU, W=layer.wgu, x=b.x, y=b.act,
              norm_w=layer.ln2, eps=cfg.rms_eps),
            J(nat.JOB_GEMV, N=cfg.hidden, K=cfg.intermediate, flags=nat.EPI_RESIDUAL, W=layer.wd, x=b.act, y=b.x, residual=b.x),
            J(nat.JOB_GEMV, N=cfg.qkv_dim, K=cfg.hidden, flags=nat.EPI_BIAS if nxt.bqkv is not None else 0, W=nxt.wqkv,
              x=b.x, y=b.qkv, bias=nxt.bqkv, norm_w=nxt.ln1, eps=cfg.rms_eps)]


def rope_tables(nat, cfg, T_max):
    d = cfg.head_dim
    inv = 1.0 / (cfg.rope_theta ** (torch.arange(0, d, 2, dtype=torch.float32, device="cuda") / d))
    return nat.rope_table(inv, T_max)


# ------------------------------------------------------------------------------------------------ GEMV-job cases
def _forms():
    from tests import linear_cases as L
    return {"plain": dict(flags=0), "bias": dict(flags=L.EPI_BIAS), "res_inplace": dict(flags=L.EPI_RESIDUAL, alias=True),
            "norm_swiglu": dict(flags=L.EPI_SWIGLU, norm=True), "norm_bias": dict(flags=L.EPI_BIAS, norm=True),
            "norm": dict(flags=0, norm=True)}


def model_gemv_jobs(cfg, rows=(1, 2, 3, 4)):
    """the four GEMV jobs of a layer's chain (ml/shard.py) as linear_cases Cases: qkv with the RMSNorm prologue (and
    bias), o and down in place on the residual, gate/up with the norm and SwiGLU"""
    from tests import linear_cases as L
    F = _forms()
    out = []
    for M in rows:
        for name, N, K, form in (("qkv", cfg.qkv_dim, cfg.hidden, "norm_bias" if cfg.qkv_bias else "norm"),
                                 ("o", cfg.hidden, cfg.q_dim, "res_inplace"), ("gu", 2 * cfg.intermediate, cfg.hidden, "norm_swiglu"),
                                 ("down", cfg.hidden, cfg.intermediate, "res_inplace")):
            kw = F[form]
            out.append(L.Case(f"chain.{cfg.name}.m{M}.{name}", "gemv", M, N, K, flags=kw["flags"],
                              alias=kw.get("alias", False), norm=kw.get("norm", False), ld_pad=0))
    return out


def edge_gemv_jobs(rows=(1, 2, 3, 4)):
    """shapes at the ring's edges for each row count, with the forms in rotation: K at the K chunk and one vector past
    it (two chunks, the second of 8 elements), K at 2 and 8 pairs per slot and one vector past, K = 8 and 24 with a
    partial last unit, and fewer units than CTAs (plain and chunked)"""
    from tests import linear_cases as L
    F = _forms()
    names = ["plain", "bias", "res_inplace", "norm_swiglu", "norm_bias"]
    out, i = [], 0
    for M in rows:
        shapes = []
        for pairs in (1, 2, 8):
            K = kc_edge(M, pairs=pairs)
            shapes += [(f"p{pairs}edge", 2 * (8 * 3 + 3), K), (f"p{pairs}edge+8", 2 * (8 * 3 + 3), K + 8)]
        shapes += [("k8", 2 * (8 * 5 + 3), 8), ("k24", 2 * (8 * 5 + 3), 24), ("few_units", 10, 512),
                   ("few_chunked", 6, kc_edge(M) + 8)]
        for tag, N, K in shapes:
            form = names[i % len(names)]
            i += 1
            kw = F[form]
            out.append(L.Case(f"chain.edge.m{M}.{tag}.{form}", "gemv", M, N, K, flags=kw["flags"],
                              alias=kw.get("alias", False), norm=kw.get("norm", False), ld_pad=0))
    return out
