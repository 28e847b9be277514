"""The weight-streaming GEMV hands out its rows by ticket from a block of device counter words (tl_gemv_bf16_ctr).
Every decode Linear shape of every config, at 1..4 rows, in the one-ring and the two-ring regime, element by element
against the float64 chain of tests/linear_cases.py with guard bands around the outputs; the counters are back at zero
after each call, after 100 graph replays and after back-to-back launches that overlap under programmatic dependent
launch; and a grid with more CTAs than units."""
from dataclasses import replace

import pytest
import torch

from tensorlink_b200.ml import configs as C
from tests import linear_cases as L

pytestmark = pytest.mark.gpu
CONFIGS = [C.QWEN25_05B, C.QWEN25_7B, C.QWEN3_8B, C.TINY_QWEN2, C.TINY_QWEN2_D128, C.TINY_QWEN3]


@pytest.fixture(scope="module")
def nat():
    from tensorlink_b200 import native
    native.require_device()
    return native


@pytest.fixture(scope="module")
def sms(nat):
    return torch.cuda.get_device_properties(0).multi_processor_count


def ctr_launch(nat, ctr):
    """launch(c, bufs) through tl_gemv_bf16_ctr with the caller's counter block"""
    lib = nat.load()

    def launch(c, bufs):
        a, b, out = bufs["a"], bufs["b"], bufs["c"]
        res = out.ptr if c.alias else (bufs["res"].ptr if "res" in bufs else None)
        nxt = bufs["next"].ptr if c.next_w else None
        rc = lib.tl_gemv_bf16_ctr(a.ptr, b.ptr, out.ptr, c.M, c.N, c.K, bufs["bias"].ptr if "bias" in bufs else None, res,
                                  bufs["g"].ptr if "g" in bufs else None, L.EPS, c.flags, ctr.data_ptr(), nxt,
                                  (8 << 20) if nxt else 0, nat._stream())
        nat._check(rc, c.name)
    return launch


def decode_cases(cfg, rows=(1, 2, 3, 4)):
    return [c for c in L.model_calls(cfg, gemv_rows=rows) if c.op == "gemv"]


@pytest.mark.parametrize("cfg", CONFIGS, ids=lambda c: c.name)
def test_decode_shapes(nat, sms, cfg):
    ctr = nat.gemv_counters(device="cuda")
    launch = ctr_launch(nat, ctr)
    errors = []
    for c in decode_cases(cfg):
        for leg in ("exact", "round"):
            if leg == "exact" and not c.exact_ok:
                continue
            errors += L.check_call(c, leg, launch, "cuda", sms)["errors"]
            torch.cuda.synchronize()
            assert int(ctr.abs().sum()) == 0, (c.name, leg, ctr.tolist())
    assert not errors, "\n".join(errors[:20])


def test_both_ring_regimes_are_covered(sms):
    regimes = set()
    for cfg in CONFIGS:
        for c in decode_cases(cfg):
            p = L.gemv_stream_params(min(c.M, 4), c.N, c.K, sms, {})
            if p:
                regimes.add((p[0], p[2]))
    assert {(1, False), (1, True), (2, False)} <= regimes, regimes


def _layer(cfg, M, gen):
    """random operands for the four decode GEMVs of one layer and the lm_head"""
    def t(*s):
        return (torch.randn(*s, generator=gen, device="cuda") * 0.05).bfloat16()
    H, I, Q, QKV, V = cfg.hidden, cfg.intermediate, cfg.q_dim, cfg.qkv_dim, cfg.vocab
    return dict(x=t(M, H), attn=t(M, Q), wqkv=t(QKV, H), wo=t(H, Q), wgu=t(2 * I, H), wd=t(H, I), head=t(V, H), g=t(H) + 1)


def _step(nat, p, ctr):
    x = p["x"].clone()
    qkv = nat.gemv(x, p["wqkv"], norm_w=p["g"], next_w=p["wo"], counter=None if ctr is None else ctr[0])
    nat.gemv(p["attn"], p["wo"], out=x, residual=x, next_w=p["wgu"], counter=None if ctr is None else ctr[1])
    act = nat.gemv(x, p["wgu"], norm_w=p["g"], flags=nat.EPI_SWIGLU, next_w=p["wd"], counter=None if ctr is None else ctr[2])
    nat.gemv(act, p["wd"], out=x, residual=x, next_w=p["head"], counter=None if ctr is None else ctr[3])
    logits = nat.gemv(x, p["head"], norm_w=p["g"], counter=None if ctr is None else ctr[4])
    return qkv, act, x, logits


@pytest.mark.parametrize("cfg,M", [(C.QWEN25_7B, 1), (C.QWEN25_05B, 3), (C.TINY_QWEN2, 4)], ids=lambda v: getattr(v, "name", v))
def test_graph_replays_give_the_same_bits(nat, cfg, M):
    gen = torch.Generator(device="cuda").manual_seed(7)
    p = _layer(cfg, M, gen)
    ctr = nat.gemv_counters(5, device="cuda")
    want = [t.clone() for t in _step(nat, p, ctr)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _step(nat, p, ctr)                         # warm-up outside the capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            outs = _step(nat, p, ctr)
    torch.cuda.current_stream().wait_stream(s)
    for i in range(100):
        g.replay()
        if i % 25 == 0 or i == 99:
            torch.cuda.synchronize()
            for a, b in zip(outs, want):
                assert torch.equal(a.view(torch.int16), b.view(torch.int16)), i
    torch.cuda.synchronize()
    assert int(ctr.abs().sum()) == 0, ctr.tolist()


def test_back_to_back_pool_launches_match_separated_ones(nat):
    """pool blocks: 60 dependent calls launched back to back (they overlap under PDL) equal the same calls with a
    synchronise after each"""
    cfg = C.QWEN25_05B
    gen = torch.Generator(device="cuda").manual_seed(11)
    p = _layer(cfg, 2, gen)

    def chain(sync):
        outs = []
        for _ in range(12):
            outs += [t.clone() for t in _step(nat, p, None)]
            if sync:
                torch.cuda.synchronize()
        torch.cuda.synchronize()
        return outs
    a, b = chain(False), chain(True)
    for u, v in zip(a, b):
        assert torch.equal(u.view(torch.int16), v.view(torch.int16))


@pytest.mark.parametrize("M", [1, 4])
def test_grid_larger_than_the_number_of_units(nat, sms, M):
    """K = 64: a unit is 8 pairs, so 64 rows are 4 units for 32 CTAs; and one pair (grid 1) on 2 rows"""
    ctr = nat.gemv_counters(device="cuda")
    launch = ctr_launch(nat, ctr)
    for N, K in ((64, 64), (2, 64), (130, 64)):
        c = L.Case(f"grid_gt_units.{N}x{K}", "gemv", M, N, K, ld_pad=0)
        per_sm, P, chunked, grid = L.gemv_stream_params(M, N, K, sms, {})
        assert grid > -(-(N // 2) // P) or N == 2, (grid, P)
        for flags in (0, L.EPI_RESIDUAL):
            for leg in ("exact", "round"):
                r = L.check_call(replace(c, flags=flags), leg, launch, "cuda", sms)
                assert not r["errors"], r["errors"][:10]
            torch.cuda.synchronize()
            assert int(ctr.abs().sum()) == 0, ctr.tolist()
