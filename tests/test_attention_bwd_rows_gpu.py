"""``tl_attn_bwd_rows``: the attention backward of a left-padded training batch (include/tensorlink_b200.h), through
both backward forms, against fp32 autograd of the masked softmax.

Row b of each case starts with ``kv_start[b]`` pad tokens: their q / dO / out / lse rows and their K/V slots are NaN,
so any read of them that does not go through a select shows up.  Real query rows and real keys are compared with the
rel-L2 bound of tests/test_train_gpu.py::test_attn_bwd.  dq, dk and dv start as NaN (training allocates them empty):
pad query rows of dq and pad slots of dk / dv must be exact zeros, and dk / dv slots past S must keep their NaN.  With
every start 0 the result must equal ``tl_attn_bwd`` bit for bit.  tests/test_attention_bwd_rows_numerics_gpu.py checks
the same entry point row by row on peaked scores."""
import pytest
import torch
import torch.nn.functional as F

from oracle import shard_oracle as O

pytestmark = pytest.mark.gpu
TOL = 4e-3          # tests/test_train_gpu.py::test_attn_bwd

SHAPES = [(2, 64, 4, 2, 64), (1, 100, 14, 2, 64), (2, 130, 4, 2, 128), (1, 257, 8, 8, 128), (2, 192, 14, 2, 64),
          (1, 200, 6, 3, 64), (2, 40, 4, 2, 128), (2, 50, 7, 1, 64)]


@pytest.fixture(scope="module")
def nat():
    from tensorlink_b200 import native
    native.require_device()
    return native


def rnd(*shape, seed=0, std=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * std).bfloat16()


def close(got, want):
    """rel-L2 <= TOL; a gradient that is 0 in exact arithmetic (dq and dk of a row whose only key is itself: the softmax
    is constant) is held to an absolute bound instead"""
    if float(want.norm()) < 1e-6:
        return float(got.float().abs().max()) <= 1e-5
    return O.rel_l2(got, want) <= TOL


def start_sets(B, S):
    """per-row starts: 0, inside the first tile, exactly one tile, inside a later tile, S - 1 (one real token), and
    mixed within a batch"""
    cands = [c for c in (0, 5, 64, 100, S - 1) if c < S]
    return [[cands[(i + j) % len(cands)] for j in range(B)] for i in range(len(cands))]


def reference(q, k, v, do, starts, scale):
    """fp32 autograd of softmax(QK^T * scale + causal + key mask) V; pad query rows (no key) output 0"""
    B, S, n_h, d = q.shape
    n_rep = n_h // k.shape[1]
    qf, kf, vf = q.float().requires_grad_(), k.float().requires_grad_(), v.float().requires_grad_()
    st = torch.tensor(starts)
    real_key = torch.arange(S)[None, :] >= st[:, None]                                   # [B,S]
    allowed = real_key[:, None, None, :] & (torch.arange(S)[None, :] <= torch.arange(S)[:, None])[None, None]
    s = (qf.transpose(1, 2) @ O.repeat_kv(kf, n_rep).transpose(2, 3)) * scale
    s = s.masked_fill(~allowed, float("-inf"))
    p = torch.where(allowed.any(-1, keepdim=True), F.softmax(s, -1), torch.zeros(()))
    of = (p.nan_to_num(0.0) @ O.repeat_kv(vf, n_rep)).transpose(1, 2).reshape(B, S, -1)
    of.backward(do.float())
    return qf.grad, kf.grad, vf.grad, real_key


def run(nat, q, kc, vc, do, B, S, n_h, n_kv, d, kv_start, poison=None):
    """forward (rows form when kv_start is given) then backward; ``poison`` (bool [B,S]) sets those rows of out and lse
    to NaN before the backward"""
    scale = d ** -0.5
    T_max = kc.shape[2]
    out = torch.empty(B, S, n_h * d, dtype=torch.bfloat16, device="cuda")
    lse = torch.empty(B, n_h, S, dtype=torch.float32, device="cuda")
    nat.attn_prefill_fwd(q, kc, vc, out, lse, B, S, 0, n_h, n_kv, d, scale, kv_start=kv_start)
    if poison is not None:
        pm = poison.cuda()
        out[pm] = float("nan")
        lse.transpose(1, 2)[pm] = float("nan")
    dq = torch.full((B, S, n_h, d), float("nan"), dtype=torch.bfloat16, device="cuda")
    dk = torch.full((B, n_h, T_max, d), float("nan"), dtype=torch.bfloat16, device="cuda")   # as training's empty buffers
    dv = torch.full_like(dk, float("nan"))
    ws = torch.empty(nat.attn_bwd_ws(B, S, n_h), dtype=torch.uint8, device="cuda")
    nat.attn_bwd(q, kc, vc, out, do, lse, dq, dk, dv, ws, B, S, n_h, n_kv, d, scale, kv_start=kv_start)
    torch.cuda.synchronize()
    return dq.cpu(), dk.cpu(), dv.cpu()


@pytest.mark.parametrize("impl", ["mma", "wgmma"])
@pytest.mark.parametrize("B,S,n_h,n_kv,d", SHAPES)
def test_attn_bwd_rows_vs_masked_autograd(nat, monkeypatch, B, S, n_h, n_kv, d, impl):
    monkeypatch.setenv("TL_ATTN_BWD", impl)
    n_rep = n_h // n_kv
    q, k, v = rnd(B, S, n_h, d, seed=12, std=0.7), rnd(B, n_kv, S, d, seed=13, std=0.7), rnd(B, n_kv, S, d, seed=14)
    do = rnd(B, S, n_h * d, seed=15)
    T_max = S + 3
    for starts in start_sets(B, S):
        gq, gk, gv, real = reference(q, k, v, do, starts, d ** -0.5)
        pad = ~real
        qn, don = q.clone(), do.clone()
        qn[pad], don[pad] = float("nan"), float("nan")
        kc = torch.zeros(B, n_kv, T_max, d, dtype=torch.bfloat16)
        vc = torch.zeros_like(kc)
        kc[:, :, :S], vc[:, :, :S] = k, v
        for b, s0 in enumerate(starts):
            kc[b, :, :s0], vc[b, :, :s0] = float("nan"), float("nan")
        ks = torch.tensor(starts, dtype=torch.int32, device="cuda")
        dq, dk, dv = run(nat, qn.cuda(), kc.cuda(), vc.cuda(), don.cuda(), B, S, n_h, n_kv, d, ks, poison=pad)
        assert bool(torch.isfinite(dq).all() and torch.isfinite(dk[:, :, :S]).all()
                    and torch.isfinite(dv[:, :, :S]).all()), starts
        assert dq[pad].abs().sum() == 0, starts
        dks = dk.float().view(B, n_kv, n_rep, T_max, d).sum(2)[:, :, :S]
        dvs = dv.float().view(B, n_kv, n_rep, T_max, d).sum(2)[:, :, :S]
        for b, s0 in enumerate(starts):
            assert dk[b, :, :s0].abs().sum() == 0 and dv[b, :, :s0].abs().sum() == 0, starts
        rq, rk = real, real[:, None, :].expand(B, n_kv, S)
        assert close(dq[rq], gq[rq]) and close(dks[rk], gk[rk]) and close(dvs[rk], gv[rk]), starts
        assert bool(torch.isnan(dk[:, :, S:]).all() and torch.isnan(dv[:, :, S:]).all())   # slots past S untouched


@pytest.mark.parametrize("impl", ["mma", "wgmma"])
@pytest.mark.parametrize("B,S,n_h,n_kv,d", SHAPES)
def test_attn_bwd_rows_zero_starts_equal_plain(nat, monkeypatch, B, S, n_h, n_kv, d, impl):
    monkeypatch.setenv("TL_ATTN_BWD", impl)
    q, k, v = rnd(B, S, n_h, d, seed=22, std=0.7), rnd(B, n_kv, S, d, seed=23, std=0.7), rnd(B, n_kv, S, d, seed=24)
    do = rnd(B, S, n_h * d, seed=25)
    kc, vc = k.cuda(), v.cuda()
    plain = run(nat, q.cuda(), kc, vc, do.cuda(), B, S, n_h, n_kv, d, None)
    rows = run(nat, q.cuda(), kc, vc, do.cuda(), B, S, n_h, n_kv, d, torch.zeros(B, dtype=torch.int32, device="cuda"))
    for a, b in zip(plain, rows):      # as bits: the slots past S hold NaN in both
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def test_attn_bwd_rows_rejects_bad_starts(nat):
    from tensorlink_b200.native import NativeError
    B, S, n_h, n_kv, d = 1, 64, 4, 2, 64
    z = torch.zeros(B, S, n_h * d, dtype=torch.bfloat16, device="cuda")
    kc = torch.zeros(B, n_kv, S, d, dtype=torch.bfloat16, device="cuda")
    lse = torch.zeros(B, n_h, S, dtype=torch.float32, device="cuda")
    ws = torch.empty(nat.attn_bwd_ws(B, S, n_h), dtype=torch.uint8, device="cuda")
    with pytest.raises(NativeError):
        nat.attn_bwd(z, kc, kc, z, z, lse, z, kc, kc, ws, B, S, n_h, n_kv, d, 0.125,
                     kv_start=torch.zeros(B, dtype=torch.int64, device="cuda"))
