"""The decode-chain kernel (csrc/decode_chain.cu) job by job, through tl_decode_chain directly.

  * GEMV jobs: the harness of tests/linear_cases.py (guard bands around every operand and output, the exact integer
    leg, the rounding leg's float64 bound) with the case as a one-job chain, at the four Linears of every config and at
    the ring's edges placed by tests/chain_cases.py.  Where tl_gemv_bf16 runs gemv_stream_kernel (torch.profiler says
    which kernel ran) the chain's output equals it bit for bit; where it runs the register kernel, the bound is the
    check.  Each case reports which of the two it passed.  These run in a fresh process (tests/chain_env_worker.py
    --gemv-paths): CUPTI tracing turned on in this process, which then runs chain kernels and graph captures, stopped
    recording kernels in later profiler sessions of the same process (tests/test_fp8_gpu.py's saw none).
  * The attention job: RoPE (+ q/k-norm) + KV append + split-KV attention on the designed score patterns of
    tests/attn_patterns.py, against float64 per row (tests/attn_patterns.check_rows with FWD_K / FWD_FLOOR), at the
    positions where the key partition changes, with NaN in the cache above pos and in the output.  The appended key
    and value equal what tl_rope_kv_fwd writes (with the q/k-norm, a key element may take the other bf16 neighbour
    where its normalised value lies within 2^-16 of a rounding tie), and every other cache slot is untouched.
  * Job lists: a full layer replayed with tl_gemv_bf16 from the chain's own attention output, three layers in one
    launch against three launches, and repeated launches eager and graph-captured.  After every launch every word of
    the sync slot is zero.
  * The settings the library reads once, in fresh processes (tests/chain_env_worker.py).
  * Model level: the dq mode bit for bit against the per-kernel path, the chain at Qwen2.5-7B and Qwen3-8B width, and
    four rows at 7B width, which the launcher cannot place (the step takes the per-kernel sequence).

Measured on an H100 80GB HBM3 (power limit in DESIGN.md's tolerance section): see there for the worst error / bound
ratios and the file's runtime.
"""
import json
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import pytest
import torch

from oracle import shard_oracle as O
from tensorlink_b200.ml import configs as C
from tensorlink_b200.ml.weights import init_state_dict, synthetic_tokens
from tests import attn_patterns as P
from tests import chain_cases as CC
from tests import linear_cases as L
from tests import rowwise_cases as R
from tests.chain_env_worker import STAGE_KB, stream_path

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAN = float("nan")
SMS_H100 = 132                     # SM count the attention cases are placed for (H100 SXM)
CONFIGS = [C.QWEN25_05B, C.QWEN25_7B, C.QWEN3_8B, C.TINY_QWEN2, C.TINY_QWEN2_D128, C.TINY_QWEN3]


@pytest.fixture(scope="module")
def nat():
    from tensorlink_b200 import native
    native.require_device()
    return native


@pytest.fixture(scope="module")
def sms(nat):
    return torch.cuda.get_device_properties(0).multi_processor_count


def bits(t):
    return t.contiguous().view(torch.int16)


# ------------------------------------------------------------------------------------------------ GEMV jobs
@pytest.fixture(scope="module")
def gemv_results(tmp_path_factory):
    """every GEMV-job group, checked in one fresh process (tests/chain_env_worker.py --gemv-paths): the torch.profiler
    session that proves which kernel tl_gemv_bf16 ran stays out of this process, which runs chain kernels and graph
    captures before and after it"""
    out = tmp_path_factory.mktemp("gemv_paths") / "res.json"
    base = {k: v for k, v in os.environ.items() if k not in ONCE_READ + ("TL_GEMV_IMPL", "TL_GEMV_CTAS_PER_SM",
                                                                         "TL_GEMV_RING_KB", "TL_GEMV_MMA")}
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "chain_env_worker.py"), str(out), "--gemv-paths"],
                       env=dict(base, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(out.read_text())


def _check_group(res, name):
    r = res[name]
    print(f"{name}: bit for bit against gemv_stream_kernel: {len(r['bits'])} cases; by the rounding bound only "
          f"(tl_gemv_bf16 runs the register kernel): {len(r['bound'])} cases {r['bound']}; refused (no ring fits): "
          f"{r['refused']}; worst |err| / bound {r['ratio']:.3f}")
    assert not r["dirty"], f"sync slot not zero after launches: {r['dirty'][:5]}"
    assert not r["errors"], "\n".join(r["errors"][:20]) + (f"\n... {len(r['errors'])} failures" if len(r["errors"]) > 20 else "")
    assert not r["path_error"], r["path_error"]
    return r


@pytest.mark.parametrize("cfg", CONFIGS, ids=lambda c: c.name)
def test_gemv_jobs_model_linears(gemv_results, sms, cfg):
    r = _check_group(gemv_results, cfg.name)
    cases = CC.model_gemv_jobs(cfg)
    # a job no ring can take beside its x (7B's down projection at four rows) is refused; every model Linear whose
    # tl_gemv_bf16 call runs gemv_stream_kernel was compared bit for bit
    assert set(r["refused"]) == {c.name for c in cases if CC.ring_geometry(c.M, c.K) is None}
    assert set(r["bits"]) == {c.name for c in cases if c.name not in r["refused"] and stream_path(c, sms)}


@pytest.mark.parametrize("M", [1, 2, 3, 4])
def test_gemv_jobs_ring_edges(gemv_results, sms, M):
    cases = CC.edge_gemv_jobs((M,))
    for c in cases:                 # the edges are where the model puts them for this geometry
        g = CC.ring_geometry(M, c.K)
        u = CC.gemv_units(c.N, c.K, g, sms)
        if ".p1edge+8." in c.name or ".few_chunked." in c.name:
            assert u["chunked"] and u["n_chunks"] == 2, c.name
        if ".p1edge." in c.name:
            assert not u["chunked"] and 4 * c.K == g["stage_bytes"], c.name
        if ".k8." in c.name or ".k24." in c.name:
            assert u["last_unit_pairs"] < u["P"], c.name
        if ".few_" in c.name:
            assert u["units"] < sms, c.name
    r = _check_group(gemv_results, f"edges.m{M}")
    assert set(r["bits"]) | set(r["bound"]) == {c.name for c in cases}


# ------------------------------------------------------------------------------------------------ attention job
_TABLES = {}
WORST = {}


def _tables_d(nat, d, T_max=CC.ATTN_T_MAX):
    key = (d, T_max)
    if key not in _TABLES:
        _TABLES[key] = nat.rope_table(1.0 / (1e6 ** (torch.arange(0, d, 2, dtype=torch.float32) / d)).cuda(), T_max)
    return _TABLES[key]


def _attn_chain(nat, qkv, kc, vc, out, posd, ct, st, qn, kn, M, n_h, n_kv, d, flags=0, eps=1e-6):
    sync = torch.zeros(nat.CHAIN_SYNC_BYTES // 4, dtype=torch.int32, device="cuda")
    ws = torch.empty(nat.decode_chain_ws(M, n_h, n_kv, d), dtype=torch.uint8, device="cuda")
    job = nat.make_job(nat.JOB_ATTN, x=qkv, y=out, k_cache=kc, v_cache=vc, pos_dev=posd, cos_tab=ct, sin_tab=st,
                       q_norm_w=qn, k_norm_w=kn, n_h=n_h, n_kv=n_kv, d=d, T_max=kc.shape[2], scale=d ** -0.5, eps=eps,
                       flags=flags)
    nat.DecodeChain([job], M, sync, ws).launch()
    torch.cuda.synchronize()
    assert not bool(sync.any()), f"sync slot words {sync.nonzero()[:8, 0].tolist()} not zero after the launch"


def _key_candidates(qkv, kn, ct, st, pos, n_h, n_kv, d, eps):
    """the bf16 values tl_rope_kv_fwd's key may take with the q/k-norm (tests/rowwise_cases.py's band): each normalised
    element within 2^-16 of a rounding tie may round either way, every (x1, x2) combination rotated as HF does"""
    M, half = qkv.shape[0], d // 2
    x = qkv.view(M, -1, d)[:, n_h:n_h + n_kv].cpu().double()
    rstd = 1.0 / torch.sqrt((x * x).mean(-1, keepdim=True) + float(torch.tensor(eps, dtype=torch.float32)))
    n64 = x * rstd
    near, other, tie = R.neighbours(n64)
    alt = torch.where(tie <= R.NORM_TIE_REL * n64.abs(), other, near)
    w = kn.cpu().double()
    y0, y1 = R.rbf(w * near), R.rbf(w * alt)
    cc, ss = ct[pos].cpu().double(), st[pos].cpu().double()
    return [R.rope_fwd_ref(torch.cat([a[..., :half], b[..., half:]], -1), cc, ss) for a in (y0, y1) for b in (y0, y1)]


def _attn_case(nat, n_h, n_kv, d, qk_norm, M, pos, pattern, eps=1e-6):
    T_max, T = CC.ATTN_T_MAX, pos + 1
    qkv, qn, kn, kc0, vc0 = (t.cuda() if t is not None else None
                             for t in P.decode_inputs(pattern, M, pos, n_h, n_kv, d, qk_norm, T_max, eps))
    ct, st = _tables_d(nat, d)
    posd = torch.tensor([pos], dtype=torch.int32, device="cuda")
    kc1, vc1 = kc0.clone(), vc0.clone()
    q = torch.empty(M, n_h * d, dtype=torch.bfloat16, device="cuda")
    nat.rope_kv_fwd(qkv, q, kc1, vc1, posd, ct, st, qn, kn, eps, 1, n_h, n_kv, d)
    kc2, vc2 = kc0.clone(), vc0.clone()
    out = torch.full((M, n_h * d), NAN, dtype=torch.bfloat16, device="cuda")
    _attn_chain(nat, qkv, kc2, vc2, out, posd, ct, st, qn, kn, M, n_h, n_kv, d, eps=eps)
    # every slot but pos untouched (NaN above pos compares by bits), the appended value exact
    others = torch.ones(T_max, dtype=torch.bool, device="cuda")
    others[pos] = False
    assert torch.equal(bits(kc2[:, :, others]), bits(kc0[:, :, others])), "key cache written outside slot pos"
    assert torch.equal(bits(vc2[:, :, others]), bits(vc0[:, :, others])), "value cache written outside slot pos"
    assert torch.equal(bits(vc2[:, :, pos]), bits(vc1[:, :, pos])), "appended value differs from tl_rope_kv_fwd's"
    flips = 0
    if qk_norm:
        errors = []
        cands = _key_candidates(qkv, kn, ct, st, pos, n_h, n_kv, d, eps)
        R.check_candidates("chain key", kc2[:, :, pos], cands, errors)
        R.check_candidates("tl_rope_kv_fwd key", kc1[:, :, pos], cands, errors)
        assert not errors, errors
        flips = int((bits(kc2[:, :, pos]) != bits(kc1[:, :, pos])).sum())
    else:
        assert torch.equal(bits(kc2[:, :, pos]), bits(kc1[:, :, pos])), "appended key differs from tl_rope_kv_fwd's"
    qr, k, v = q.view(M, 1, n_h, d), kc1[:, :, :T], vc1[:, :, :T]
    ref, _ = P.ref_fwd(qr, k, v, pos, d ** -0.5)
    ratio = P.check_rows(f"{pattern} pos={pos} out", out.view(M, 1, n_h, d), ref, P.oracle_fwd(qr, k, v, d ** -0.5),
                         P.FWD_K, P.FWD_FLOOR)
    WORST["attn"] = max(WORST.get("attn", 0.0), ratio)
    return ratio, flips


def _attn_id(c):
    n_h, n_kv, d, qn, M, pos, pat = c
    return f"h{n_h}kv{n_kv}d{d}{'n' if qn else ''}-m{M}-pos{pos}-{pat}"


@pytest.mark.parametrize("case", CC.attn_cases(SMS_H100), ids=_attn_id)
def test_attention_job(nat, sms, case):
    n_h, n_kv, d, qk_norm, M, pos, pattern = case
    ratio, flips = _attn_case(nat, n_h, n_kv, d, qk_norm, M, pos, pattern)
    part = CC.attn_partition(sms, n_kv, M, pos)
    print(f"{_attn_id(case)}: {part['cpg_eff']} CTAs of {part['chunk']} keys, |err| / bound {ratio:.3f}, "
          f"key flips {flips}; worst so far {WORST['attn']:.3f}")


@pytest.mark.parametrize("n_h,n_kv,d,qk_norm", [(28, 4, 128, False), (32, 8, 128, True), (14, 2, 64, True)])
def test_pos_per_row_same_position_changes_no_bit(nat, n_h, n_kv, d, qk_norm):
    M, pos, eps = 3, 700, 1e-6
    qkv, qn, kn, kc0, vc0 = (t.cuda() if t is not None else None
                             for t in P.decode_inputs("rising", M, pos, n_h, n_kv, d, qk_norm, 1024, eps))
    ct, st = _tables_d(nat, d)
    res = []
    for flags, posd in ((0, torch.tensor([pos], dtype=torch.int32)), (nat.ATTN_POS_PER_ROW, torch.full((M,), pos, dtype=torch.int32))):
        kc, vc = kc0.clone(), vc0.clone()
        out = torch.full((M, n_h * d), NAN, dtype=torch.bfloat16, device="cuda")
        _attn_chain(nat, qkv, kc, vc, out, posd.cuda(), ct, st, qn, kn, M, n_h, n_kv, d, flags=flags, eps=eps)
        res.append([bits(t) for t in (out, kc, vc)])
    assert all(torch.equal(a, b) for a, b in zip(*res))


@pytest.mark.parametrize("n_h,n_kv,d,qk_norm,positions", [
    (14, 2, 64, True, (0, 127, 128, 3000)), (28, 4, 128, False, (5, 300, 8191)), (32, 8, 128, True, (2047, 31))])
def test_pos_per_row_distinct_positions(nat, n_h, n_kv, d, qk_norm, positions):
    """each row at its own position meets the float64 criterion there (rows built one by one, each its own pattern)"""
    M, eps, T_max = len(positions), 1e-6, CC.ATTN_T_MAX
    pats = ["spike@T-1", "rising", "sink", "wide"]
    rows = [P.decode_inputs(pats[b], 1, p, n_h, n_kv, d, qk_norm, T_max, eps, seed=51 + b) for b, p in enumerate(positions)]
    qkv = torch.cat([r[0] for r in rows]).cuda()
    qn, kn = rows[0][1], rows[0][2]
    if qk_norm:      # one gain per layer: the rows' designed new keys follow row 0's gain, the criterion is per row anyway
        qn, kn = qn.cuda(), kn.cuda()
    kc0, vc0 = torch.cat([r[3] for r in rows]).cuda(), torch.cat([r[4] for r in rows]).cuda()
    ct, st = _tables_d(nat, d)
    posd = torch.tensor(positions, dtype=torch.int32, device="cuda")
    kc, vc = kc0.clone(), vc0.clone()
    out = torch.full((M, n_h * d), NAN, dtype=torch.bfloat16, device="cuda")
    _attn_chain(nat, qkv, kc, vc, out, posd, ct, st, qn, kn, M, n_h, n_kv, d, flags=nat.ATTN_POS_PER_ROW, eps=eps)
    for b, pos in enumerate(positions):
        kc1, vc1 = kc0[b:b + 1].clone(), vc0[b:b + 1].clone()
        q = torch.empty(1, n_h * d, dtype=torch.bfloat16, device="cuda")
        nat.rope_kv_fwd(qkv[b:b + 1].contiguous(), q, kc1, vc1, posd[b:b + 1], ct, st, qn, kn, eps, 1, n_h, n_kv, d)
        assert torch.equal(bits(vc[b:b + 1]), bits(vc1)), f"row {b}: value cache differs from tl_rope_kv_fwd's"
        if not qk_norm:
            assert torch.equal(bits(kc[b:b + 1]), bits(kc1)), f"row {b}: key cache differs from tl_rope_kv_fwd's"
        qr, k, v = q.view(1, 1, n_h, d), kc1[:, :, :pos + 1], vc1[:, :, :pos + 1]
        ref, _ = P.ref_fwd(qr, k, v, pos, d ** -0.5)
        P.check_rows(f"row {b} pos={pos}", out[b:b + 1].view(1, 1, n_h, d), ref, P.oracle_fwd(qr, k, v, d ** -0.5),
                     P.FWD_K, P.FWD_FLOOR)


# ------------------------------------------------------------------------------------------------ job lists
def _layer_setup(nat, cfg, M, pos, T_max, n_layers=1, seed=11):
    layers = [CC.ChainLayer(cfg, M, pos, T_max, seed + i) for i in range(n_layers + 1)]      # + the next layer's qkv
    b = CC.ChainBufs(cfg, M)
    g = torch.Generator(device="cuda").manual_seed(seed)
    b.x.copy_(torch.randn(M, cfg.hidden, generator=g, device="cuda"))
    b.qkv.copy_(torch.randn(M, cfg.qkv_dim, generator=g, device="cuda"))
    b.attn.fill_(NAN)
    b.act.fill_(NAN)
    ct, st = CC.rope_tables(nat, cfg, T_max)
    posd = torch.tensor([pos], dtype=torch.int32, device="cuda")
    sync = torch.zeros(2, nat.CHAIN_SYNC_BYTES // 4, dtype=torch.int32, device="cuda")
    ws = torch.empty(nat.decode_chain_ws(M, cfg.n_heads, cfg.n_kv_heads, cfg.head_dim), dtype=torch.uint8, device="cuda")
    return layers, b, ct, st, posd, sync, ws


LAYER_CASES = [(C.TINY_QWEN2, M) for M in (1, 2, 3, 4)] + [(C.TINY_QWEN3, 3), (C.QWEN25_05B, 1), (C.QWEN25_05B, 4),
                                                          (C.QWEN25_7B, 1), (C.QWEN25_7B, 3), (C.QWEN3_8B, 2)]


@pytest.mark.parametrize("cfg,M", LAYER_CASES, ids=lambda v: v.name if hasattr(v, "name") else f"m{v}")
def test_full_layer_equals_gemv_replay(nat, sms, cfg, M):
    """[ATTN, o, gate/up, down, qkv(next)] in one launch; the four GEMVs replayed with tl_gemv_bf16 from the chain's own
    attention output and the saved x give the same act, x and qkv bit for bit (the cross-CTA dependencies and the
    L2-coherent staging of data other CTAs wrote)"""
    pos, T_max = 300, 512
    (lay, nxt), b, ct, st, posd, sync, ws = _layer_setup(nat, cfg, M, pos, T_max)
    x0 = b.x.clone()
    nat.DecodeChain(CC.layer_jobs(nat, cfg, lay, nxt, b, posd, ct, st, T_max), M, sync[0], ws).launch()
    torch.cuda.synchronize()
    assert not bool(sync.any())
    assert bool(torch.isfinite(b.attn.float()).all())
    for N, K in ((cfg.hidden, cfg.q_dim), (2 * cfg.intermediate, cfg.hidden), (cfg.hidden, cfg.intermediate), (cfg.qkv_dim, cfg.hidden)):
        assert stream_path(L.Case("replay", "gemv", M, N, K), sms), (N, K)       # the replay runs gemv_stream_kernel
    x = x0.clone()
    nat.gemv(b.attn, lay.wo, out=x, residual=x)
    act = nat.gemv(x, lay.wgu, norm_w=lay.ln2, eps=cfg.rms_eps, flags=nat.EPI_SWIGLU)
    nat.gemv(act, lay.wd, out=x, residual=x)
    qkv = nat.gemv(x, nxt.wqkv, bias=nxt.bqkv, norm_w=nxt.ln1, eps=cfg.rms_eps)
    for name, a, r in (("act", b.act, act), ("x", b.x, x), ("qkv", b.qkv, qkv)):
        assert torch.equal(bits(a), bits(r)), f"{name}: {int((bits(a) != bits(r)).sum())} of {a.numel()} differ"


@pytest.mark.parametrize("cfg,M", [(C.TINY_QWEN2, 2), (C.TINY_QWEN3, 3), (C.QWEN25_05B, 1)], ids=lambda v: getattr(v, "name", f"m{v}"))
def test_three_layers_in_one_launch_equal_three_launches(nat, cfg, M):
    pos, T_max = 200, 256
    runs = []
    for per in (3, 1):
        layers, b, ct, st, posd, sync, ws = _layer_setup(nat, cfg, M, pos, T_max, n_layers=3)
        jobs = [CC.layer_jobs(nat, cfg, layers[i], layers[i + 1], b, posd, ct, st, T_max) for i in range(3)]
        if per == 3:
            nat.DecodeChain(jobs[0] + jobs[1] + jobs[2], M, sync[0], ws).launch()
        else:
            for i in range(3):
                nat.DecodeChain(jobs[i], M, sync[i % 2], ws).launch()
        torch.cuda.synchronize()
        assert not bool(sync.any())
        runs.append([bits(t) for t in b.state()] + [bits(l.kc[:, :, pos]) for l in layers[:3]] +
                    [bits(l.vc[:, :, pos]) for l in layers[:3]])
    assert all(torch.equal(a, c) for a, c in zip(*runs))


def _private_chains(nat, cfg, M, n, pos, T_max):
    """n launch sites of one layer, each with its own outputs and sync slot, all reading the same inputs (no job writes
    what another reads), so every launch can be compared with the first"""
    (lay, nxt), b, ct, st, posd, sync, ws = _layer_setup(nat, cfg, M, pos, T_max)
    J, bf = nat.make_job, torch.bfloat16
    slots = torch.zeros(n, nat.CHAIN_SYNC_BYTES // 4, dtype=torch.int32, device="cuda")
    outs, chains = [], []
    for i in range(n):
        o = {k: torch.full((M, w), NAN, dtype=bf, device="cuda") for k, w in
             (("attn", cfg.q_dim), ("x1", cfg.hidden), ("act", cfg.intermediate), ("x2", cfg.hidden), ("qkv", cfg.qkv_dim))}
        jobs = [CC.layer_jobs(nat, cfg, lay, nxt, b, posd, ct, st, T_max)[0],
                J(nat.JOB_GEMV, N=cfg.hidden, K=cfg.q_dim, flags=nat.EPI_RESIDUAL, W=lay.wo, x=o["attn"], y=o["x1"], residual=b.x),
                J(nat.JOB_GEMV, N=2 * cfg.intermediate, K=cfg.hidden, flags=nat.EPI_SWIGLU, W=lay.wgu, x=o["x1"], y=o["act"],
                  norm_w=lay.ln2, eps=cfg.rms_eps),
                J(nat.JOB_GEMV, N=cfg.hidden, K=cfg.intermediate, flags=nat.EPI_RESIDUAL, W=lay.wd, x=o["act"], y=o["x2"],
                  residual=o["x1"]),
                J(nat.JOB_GEMV, N=cfg.qkv_dim, K=cfg.hidden, flags=nat.EPI_BIAS if nxt.bqkv is not None else 0, W=nxt.wqkv,
                  x=o["x2"], y=o["qkv"], bias=nxt.bqkv, norm_w=nxt.ln1, eps=cfg.rms_eps)]
        jobs[0].y = o["attn"].data_ptr()
        outs.append(o)
        chains.append(nat.DecodeChain(jobs, M, slots[i], ws, nxt.wqkv))
    chains[0].keep = (lay, nxt, b, ct, st, posd, sync, ws)      # the job lists hold raw pointers into these
    return chains, outs, slots


@pytest.mark.parametrize("cfg,M", [(C.TINY_QWEN2_D128, 2), (C.QWEN25_05B, 1), (C.QWEN25_7B, 3)], ids=lambda v: getattr(v, "name", f"m{v}"))
def test_repeated_launches_eager_and_graph_give_the_same_bits(nat, cfg, M):
    n, pos, T_max = 6, 400, 512
    chains, outs, slots = _private_chains(nat, cfg, M, n, pos, T_max)
    for ch in chains:               # back to back on one stream
        ch.launch()
    torch.cuda.synchronize()
    assert not bool(slots.any()), f"sync words not zero after the eager launches: {slots.nonzero()[:8].tolist()}"
    first = {k: bits(v).clone() for k, v in outs[0].items()}
    assert all(bool(torch.isfinite(v.float()).all()) for v in outs[0].values())
    for i, o in enumerate(outs):
        for k, v in o.items():
            assert torch.equal(bits(v), first[k]), f"eager launch {i}: {k} differs from launch 0"
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side), torch.cuda.graph(graph, stream=side):
        for ch in chains:
            ch.launch()
    torch.cuda.current_stream().wait_stream(side)
    for rep in range(2):
        for o in outs:
            for v in o.values():
                v.fill_(NAN)
        graph.replay()
        torch.cuda.synchronize()
        assert not bool(slots.any()), f"sync words not zero after graph replay {rep}"
        for i, o in enumerate(outs):
            for k, v in o.items():
                assert torch.equal(bits(v), first[k]), f"graph replay {rep}, launch {i}: {k} differs from the eager bits"


# ------------------------------------------------------------------------------------------------ once-read settings
SETTINGS = dict({"default": {}, "dynamic": {"TL_CHAIN_DYNAMIC": "1"}, "l2ahead": {"TL_CHAIN_L2_AHEAD_KB": "512"},
                 "nopdl": {"TL_PDL": "0"}}, **{name: {"TL_CHAIN_STAGE_KB": str(kb)} for name, kb in STAGE_KB.items()})
ONCE_READ = ("TL_CHAIN_STAGE_KB", "TL_CHAIN_DYNAMIC", "TL_CHAIN_L2_AHEAD_KB", "TL_PDL")


def test_settings_read_once_give_the_same_bits(tmp_path):
    """each setting in a fresh process: the GEMV-job set and a full 0.5B-width layer give the default's bits"""
    base = {k: v for k, v in os.environ.items() if k not in ONCE_READ}

    def one(name):
        return subprocess.run([sys.executable, os.path.join(ROOT, "tests", "chain_env_worker.py"), str(tmp_path / f"{name}.json")],
                              env=dict(base, PYTHONPATH=ROOT, **SETTINGS[name]), capture_output=True, text=True, timeout=600,
                              cwd=ROOT)

    with ThreadPoolExecutor(4) as ex:
        runs = dict(zip(SETTINGS, ex.map(one, SETTINGS)))
    results = {}
    for name, r in runs.items():
        assert r.returncode == 0, (name, r.stderr[-3000:])
        res = json.loads((tmp_path / f"{name}.json").read_text())
        assert not res["errors"], (name, res["errors"][:10])
        assert not res["dirty"], (name, res["dirty"][:5])
        results[name] = res
        print(name, "geometry of the 0.5B layer (M/K_max: slot bytes, slots, NW, K chunk):", res["geometry"])
    for name, kb in STAGE_KB.items():
        assert results[name]["geometry"]["1/4864"][2] == CC.ring_geometry(1, 4864, kb)["NW"], name
    ref = results["default"]["bits"]
    for name, res in results.items():
        common = set(ref) & set(res["bits"])
        assert {k for k in ref if k.startswith("layer/")} <= common, name
        diff = sorted(k for k in common if res["bits"][k] != ref[k])
        assert not diff, (name, diff[:10])


# ------------------------------------------------------------------------------------------------ model level
def _dm(cfg, monkeypatch, impl, **kw):
    from tensorlink_b200.ml import DistributedModel
    monkeypatch.setenv("TL_DECODE_IMPL", impl)
    kw.setdefault("max_seq", 128)
    return DistributedModel(cfg, training=False, **kw)


def _decode_logits(dm, ids, steps, use_graph=True):
    st = dm.stage
    B, S = ids.shape
    st.prefill(st.embed(ids[:, :S - steps].cuda()), 0, 0)
    out = []
    for s in range(steps):
        st.ids_dec[0][:B].copy_(ids[:, S - steps + s].cuda())
        st.decode(0, B, use_graph=use_graph and s % 2 == 1)
        out.append(st.logits_dec[:B].clone())
    st.check()
    return torch.stack(out).cpu()


@pytest.mark.parametrize("cfg", [C.TINY_QWEN2, C.TINY_QWEN2_D128, C.TINY_QWEN3], ids=lambda c: c.name)
@pytest.mark.parametrize("B", [1, 2, 3])
def test_dq_mode_is_bit_identical_to_the_kernel_sequence(cfg, B, monkeypatch):
    """dq runs down(j) + qkv(j+1) as a two-job chain; both jobs are gemv_stream_kernel's arithmetic"""
    ids = synthetic_tokens(cfg, B, 40)
    dq = _dm(cfg, monkeypatch, "dq", max_batch=B)
    assert dq.stage.slots[0].dq_ok(B)
    a = _decode_logits(dq, ids, 6)
    k = _dm(cfg, monkeypatch, "kernels", max_batch=B)
    b = _decode_logits(k, ids, 6)
    assert torch.equal(bits(a), bits(b))
    assert torch.equal(dq.generate(ids[:, :24], max_new_tokens=16), k.generate(ids[:, :24], max_new_tokens=16))


@pytest.mark.parametrize("base", [C.QWEN25_7B, C.QWEN3_8B], ids=lambda c: c.name)
def test_full_width_layer_chain(base, monkeypatch):
    """one full-width layer (the chunked down projection, and the 16 KB-slot ring at three rows): the chain against the
    per-kernel path and the CPU oracle under tests/test_decode_chain_gpu.py's criteria, B = 1..3"""
    cfg = base.scaled(name=base.name + "-1layer", n_layers=1)
    steps, S = 4, 24
    ids3 = synthetic_tokens(cfg, 3, S)
    sd = init_state_dict(cfg)
    with torch.no_grad():
        full16 = O.OracleModel(cfg, sd, "sdpa_math").logits(ids3)
        full32 = O.OracleModel(cfg, {k: v.float() for k, v in sd.items()}, "sdpa_math").logits(ids3)
    del sd
    chain = _dm(cfg, monkeypatch, "chain", max_batch=3)
    kern = _dm(cfg, monkeypatch, "kernels", max_batch=3)
    for B in (1, 2, 3):
        ids = ids3[:B]
        monkeypatch.setenv("TL_DECODE_IMPL", "chain")
        assert chain.stage.slots[0].chain_ok(B)
        lc = _decode_logits(chain, ids, steps, use_graph=False)
        monkeypatch.setenv("TL_DECODE_IMPL", "kernels")
        lk = _decode_logits(kern, ids, steps, use_graph=False)
        ref16 = full16[:B, S - steps:S].transpose(0, 1)
        ref32 = full32[:B, S - steps:S].transpose(0, 1)
        e_ref = O.rel_l2(ref16, ref32)
        e_chain, mutual = O.rel_l2(lc, ref32), O.rel_l2(lc, lk)
        print(f"{cfg.name} B={B}: chain-vs-fp32 {e_chain:.3e} oracle_bf16-vs-fp32 {e_ref:.3e} chain-vs-kernels {mutual:.3e}")
        assert e_chain <= 1.25 * e_ref and O.rel_l2(lc, ref16) <= 2.0 * e_ref
        assert mutual <= 2.0 * e_ref


def test_four_rows_at_7b_width_take_the_kernel_sequence(monkeypatch):
    """With TL_GEMV_MAX_ROWS=4, four rows at Qwen2.5-7B width leave 3 ring slots of 16 KB beside the staged x
    (175,488 B): the launcher refuses the shape, so chain_ok and dq_ok must too; the steps then equal the per-kernel
    sequence bit for bit.  Three rows still take the chain."""
    from tensorlink_b200.ml import shard
    monkeypatch.setenv("TL_GEMV_MAX_ROWS", "4")
    monkeypatch.setattr(shard, "_GEMV_MAX_ROWS", None)
    cfg = C.QWEN25_7B.scaled(name="Qwen2.5-7B-2layer", n_layers=2)
    ids = synthetic_tokens(cfg, 4, 20)
    dm = _dm(cfg, monkeypatch, "kernels", max_batch=4, max_seq=64, init="device")
    grp = dm.stage.slots[0]
    ref = _decode_logits(dm, ids, 3, use_graph=False)
    for impl in ("chain", "dq"):
        monkeypatch.setenv("TL_DECODE_IMPL", impl)
        assert (grp.chain_ok(3) if impl == "chain" else grp.dq_ok(3))
        assert not grp.chain_ok(4) and not grp.dq_ok(4)
        got = _decode_logits(dm, ids, 3, use_graph=False)
        assert torch.equal(bits(got), bits(ref)), impl
