"""The ordered row reductions of the backward pass, checked exactly, for accuracy and run to run.

Norm-gain, q/k-norm-gain, bias and loss reductions write one partial row per CTA (or per 256-row slab, or per CE row)
and ``det_reduce_kernel`` adds those rows in order; the embedding backward adds all tokens that share an id in token
order.  Each kernel is checked three ways:

  * exact: inputs chosen so that every term and every partial sum is representable in fp32, so the result equals
    the float64 sum bit for bit whatever the summation order.  A dropped, duplicated or misplaced partial row fails;
  * accuracy: random inputs against a float64 (or fp32-autograd) reference;
  * run to run: two calls on the same inputs from the same non-zero accumulator give the same bits.

Row counts are chosen on both sides of the grid caps, which depend on the SM count of the device, so that the loops
in which warps stride over rows and items run.
"""
import pytest
import torch
import torch.nn.functional as F

from oracle import shard_oracle as O

pytestmark = pytest.mark.gpu
TOL = 4e-3          # one bf16 rounding of a gradient output, as in tests/test_train_gpu.py


@pytest.fixture(scope="module")
def nat():
    from tensorlink_b200 import native
    native.require_device()
    return native


@pytest.fixture(scope="module")
def sms(nat):
    return torch.cuda.get_device_properties(0).multi_processor_count


def rnd(*shape, seed=0, std=1.0, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * std).to(dtype)


def rint(*shape, seed=0, lo=-4, hi=4):
    """integer-valued bf16 in [lo, hi]"""
    g = torch.Generator().manual_seed(seed)
    return torch.randint(lo, hi + 1, shape, generator=g).to(torch.bfloat16)


def acc0(n, seed=0):
    """a non-zero fp32 accumulator whose values are exact halves (the reduce does acc += sum)"""
    g = torch.Generator().manual_seed(seed)
    return torch.randint(-8, 9, (n,), generator=g).double() + 0.5


def resolve_rows(spec, sms):
    """row counts relative to the grid cap: the warp kernels run at most 4 x SMs CTAs of 4 warps"""
    cap = 4 * 4 * sms
    return {"cap-1": cap - 1, "cap+1": cap + 1}.get(spec, spec)


# ------------------------------------------------------------------------------------------------ rmsnorm_bwd
NB_H = [256, 1024, 1032, 3584]          # 1024: the widest row the warp kernel takes; 1032: the first block-kernel row
NB_ROWS = [1, 3, "cap-1", "cap+1", 8192]


@pytest.mark.parametrize("rows", NB_ROWS, ids=str)
@pytest.mark.parametrize("H", NB_H)
def test_rmsnorm_bwd_dw_exact(nat, sms, H, rows):
    """rstd = 1 and small-integer x, dy: dw = sum dy*x is exact in fp32, so any order gives the float64 sum."""
    rows = resolve_rows(rows, sms)
    x, dy = rint(rows, H, seed=1), rint(rows, H, seed=2)
    w = (1 + 0.1 * rnd(H, seed=6).float()).bfloat16()
    rstd = torch.ones(rows, dtype=torch.float32, device="cuda")
    a0 = acc0(H, seed=3)
    want = (a0 + (dy.double() * x.double()).sum(0)).float()
    assert torch.equal(want.double(), a0 + (dy.double() * x.double()).sum(0))      # the reference itself is exact
    dx = torch.empty(rows, H, dtype=torch.bfloat16, device="cuda")
    got = []
    for _ in range(2):
        dw = a0.float().cuda()
        nat.rmsnorm_bwd(x.cuda(), w.cuda(), dy.cuda(), rstd, dx, dw)
        got.append(dw.cpu())
    assert torch.equal(got[0], want)
    assert torch.equal(got[1], got[0])


@pytest.mark.parametrize("rows", NB_ROWS, ids=str)
@pytest.mark.parametrize("H", NB_H)
def test_rmsnorm_bwd_random(nat, sms, H, rows):
    """true rstd: dx against fp32 autograd, dw against float64 sum dy*bf16(x*rstd) (the kernel rounds the
    normalised value to bf16 before the product, as the forward does), and the same bits on a second call."""
    rows = resolve_rows(rows, sms)
    x, dy = rnd(rows, H, seed=4, std=2.0), rnd(rows, H, seed=5)
    w = (1 + 0.1 * rnd(H, seed=6).float()).bfloat16()
    xf, wf = x.float().requires_grad_(), w.float().requires_grad_()
    O.rmsnorm(xf, wf, 1e-6).backward(dy.float())
    rstd = torch.rsqrt(x.float().pow(2).mean(-1) + 1e-6)
    n = (x.float() * rstd[:, None]).bfloat16().double()
    a0 = acc0(H, seed=7)
    want = a0 + (dy.double() * n).sum(0)
    outs = []
    for _ in range(2):
        dx = torch.empty(rows, H, dtype=torch.bfloat16, device="cuda")
        dw = a0.float().cuda()
        nat.rmsnorm_bwd(x.cuda(), w.cuda(), dy.cuda(), rstd.cuda(), dx, dw)
        outs.append((dx.cpu(), dw.cpu()))
    (dx, dw), (dx2, dw2) = outs
    assert O.rel_l2(dx, xf.grad) <= TOL
    assert O.rel_l2(dw - a0, want - a0) <= 1e-5
    assert torch.equal(dx2, dx) and torch.equal(dw2, dw)


# ------------------------------------------------------------------------------------------------ colsum
@pytest.mark.parametrize("N", [2, 64, 66, 1152, 4608])
@pytest.mark.parametrize("M", [1, 255, 256, 257, 4097])                  # 1, 1, 1, 2 and 17 slabs of 256 rows
def test_colsum(nat, M, N):
    a0 = acc0(N, seed=8)
    dyi = rint(M, N, seed=9, lo=-8, hi=8)
    want = a0 + dyi.double().sum(0)
    got = []
    for _ in range(2):
        acc = a0.float().cuda()
        nat.colsum(dyi.cuda(), acc)
        got.append(acc.cpu())
    assert torch.equal(got[0].double(), want)
    assert torch.equal(got[1], got[0])
    dy = rnd(M, N, seed=10)
    acc = a0.float().cuda()
    nat.colsum(dy.cuda(), acc)
    assert O.rel_l2(acc.cpu() - a0, dy.double().sum(0)) <= 1e-5


@pytest.mark.parametrize("M,N", [(257, 66), (4097, 1152)])
def test_colsum_strided(nat, M, N):
    """dy is a column slice of a wider tensor (ld > N), as the bias gradient reads the q/k/v columns of dqkv."""
    wide = rint(M, N + 6, seed=11, lo=-8, hi=8)
    dy = wide[:, 2:N + 2]
    a0 = acc0(N, seed=12)
    acc = a0.float().cuda()
    dy_dev = wide.cuda()[:, 2:N + 2]
    assert dy_dev.stride(0) == N + 6
    nat.colsum(dy_dev, acc)
    assert torch.equal(acc.cpu().double(), a0 + dy.double().sum(0))


# ------------------------------------------------------------------------------------------------ qk_norm_bwd
QK_CASES = [(64, 14, 2), (128, 4, 2)]            # (d, n_h, n_kv): GQA groups of 7 and 2
QK_TOKENS = [1, 7, 600, 4096]                    # 4096 x (n_h + n_kv) items: far past the grid cap, warps stride


def _qk_call(nat, pre, dqkv, qn, kn, a_q, a_k, eps, n_h, n_kv, d):
    dq_acc, dk_acc = a_q.float().cuda(), a_k.float().cuda()
    out = dqkv.cuda()
    nat.qk_norm_bwd(pre.cuda(), out, qn.cuda(), kn.cuda(), dq_acc, dk_acc, eps, n_h, n_kv, d)
    return out.cpu(), dq_acc.cpu(), dk_acc.cpu()


@pytest.mark.parametrize("n_tok", QK_TOKENS)
@pytest.mark.parametrize("d,n_h,n_kv", QK_CASES)
def test_qk_norm_bwd_random(nat, d, n_h, n_kv, n_tok):
    heads = n_h + 2 * n_kv
    pre, dqkv = rnd(n_tok, heads * d, seed=13, std=1.5), rnd(n_tok, heads * d, seed=14)
    qn, kn = (1 + 0.1 * rnd(d, seed=15).float()).bfloat16(), (1 + 0.1 * rnd(d, seed=16).float()).bfloat16()
    eps = 1e-6
    a_q, a_k = acc0(d, seed=17), acc0(d, seed=18)
    got, gq, gk = _qk_call(nat, pre, dqkv, qn, kn, a_q, a_k, eps, n_h, n_kv, d)
    got2, gq2, gk2 = _qk_call(nat, pre, dqkv, qn, kn, a_q, a_k, eps, n_h, n_kv, d)
    assert torch.equal(got2, got) and torch.equal(gq2, gq) and torch.equal(gk2, gk)
    x, dy, o = pre.view(n_tok, heads, d), dqkv.view(n_tok, heads, d), got.view(n_tok, heads, d)
    for sl, w, a, g in ((slice(0, n_h), qn, a_q, gq), (slice(n_h, n_h + n_kv), kn, a_k, gk)):
        xf, wf = x[:, sl].float().requires_grad_(), w.float().requires_grad_()
        O.rmsnorm(xf, wf, eps).backward(dy[:, sl].float())
        assert O.rel_l2(o[:, sl], xf.grad) <= TOL
        # float64 sum of dy * bf16(x * rstd); the kernel's fp32 rstd may differ from torch's by an ulp, which can move
        # an occasional bf16(x * rstd) by one bf16 ulp, hence 1e-3 rather than fp32 rounding (the exact test pins the sum)
        rstd = torch.rsqrt(x[:, sl].float().pow(2).mean(-1, keepdim=True) + eps)
        n = (x[:, sl].float() * rstd).bfloat16().double()
        want = (dy[:, sl].double() * n).sum((0, 1))
        assert O.rel_l2(g.double() - a, want) <= 1e-3
    assert torch.equal(o[:, n_h + n_kv:], dy[:, n_h + n_kv:])       # v is not touched


@pytest.mark.parametrize("n_tok", QK_TOKENS)
@pytest.mark.parametrize("d,n_h,n_kv", QK_CASES)
def test_qk_norm_bwd_gains_exact(nat, d, n_h, n_kv, n_tok):
    """pre-norm q/k entries +-1 with eps 1e-6: bf16(x*rstd) = +-1 exactly, so with integer dy each gain gradient is an
    exact integer sum.  q and k gradients take different value ranges so that a swap of the q/k halves of a partial
    row shows."""
    heads = n_h + 2 * n_kv
    g = torch.Generator().manual_seed(19)
    sign = (torch.randint(0, 2, (n_tok, heads, d), generator=g) * 2 - 1).to(torch.bfloat16)
    pre = sign.clone()
    pre[:, n_h + n_kv:] = rnd(n_tok, n_kv, d, seed=20)
    dy = torch.cat([rint(n_tok, n_h, d, seed=21, lo=-3, hi=3), rint(n_tok, n_kv, d, seed=22, lo=-12, hi=8),
                    rnd(n_tok, n_kv, d, seed=23)], dim=1)
    qn, kn = (1 + 0.1 * rnd(d, seed=24).float()).bfloat16(), (1 + 0.1 * rnd(d, seed=25).float()).bfloat16()
    a_q, a_k = acc0(d, seed=26), acc0(d, seed=27)
    got, gq, gk = _qk_call(nat, pre.reshape(n_tok, -1), dy.reshape(n_tok, -1), qn, kn, a_q, a_k, 1e-6, n_h, n_kv, d)
    s = sign.double() * dy.double()
    assert torch.equal(gq.double(), a_q + s[:, :n_h].sum((0, 1)))
    assert torch.equal(gk.double(), a_k + s[:, n_h:n_h + n_kv].sum((0, 1)))
    assert torch.equal(got.view(n_tok, heads, d)[:, n_h + n_kv:], dy[:, n_h + n_kv:])


# ------------------------------------------------------------------------------------------------ ce_fwd_bwd
def _ce_ref(logits, labels, V):
    ok = (labels >= 0) & (labels < V)
    lse = torch.logsumexp(logits.double(), -1)
    lab = logits.double().gather(1, labels.clamp(0, V - 1)[:, None])[:, 0]
    return float(((lse - lab) * ok).sum()), int(ok.sum())


@pytest.mark.parametrize("V", [1000, 4096])
@pytest.mark.parametrize("M", [1, 2048, 2052])
def test_ce_loss_sum(nat, M, V):
    """loss against a float64 logsumexp, n_valid exactly, dlogits against fp32 autograd; rows labelled -100 or V are
    ignored; two calls into one loss_sum (as the chunked lm_head + CE does) add up."""
    logits = rnd(M, V, seed=28, std=2.0)
    g = torch.Generator().manual_seed(29)
    labels = torch.randint(0, V, (M,), generator=g)
    if M > 1:
        labels[torch.randint(0, M, (M // 10,), generator=g)] = -100
        labels[torch.randint(0, M, (M // 20,), generator=g)] = V
        labels[-1] = V
    want, n_ok = _ce_ref(logits, labels, V)
    inv_n = 1.0 / n_ok
    lf = logits.float().requires_grad_()
    (F.cross_entropy(lf, labels.masked_fill(labels == V, -100), ignore_index=-100, reduction="sum") * inv_n).backward()
    outs = []
    for _ in range(2):
        ls = torch.full((1,), 0.75, dtype=torch.float32, device="cuda")
        nv = torch.full((1,), 3, dtype=torch.int32, device="cuda")
        d = torch.empty(M, V, dtype=torch.bfloat16, device="cuda")
        nat.ce_fwd_bwd(logits.cuda(), labels.cuda(), ls, nv, d, inv_n)
        outs.append((float(ls), int(nv), d.cpu()))
    (ls, nv, d), (ls2, nv2, d2) = outs
    assert ls2 == ls and nv2 == nv and torch.equal(d2, d)
    assert nv == 3 + n_ok
    assert abs((ls - 0.75) - want) <= 1e-5 * abs(want)
    assert O.rel_l2(d, lf.grad) <= TOL
    ign = (labels < 0) | (labels >= V)
    assert float(d[ign].float().abs().sum()) == 0.0
    # chunked: two calls into one loss_sum equal the float64 total
    h = M // 2
    ls = torch.full((1,), 0.75, dtype=torch.float32, device="cuda")
    nv = torch.zeros(1, dtype=torch.int32, device="cuda")
    for a, e in ((0, h), (h, M)):
        if e > a:
            nat.ce_fwd_bwd(logits[a:e].contiguous().cuda(), labels[a:e].contiguous().cuda(), ls, nv,
                           torch.empty(e - a, V, dtype=torch.bfloat16, device="cuda"), inv_n)
    assert int(nv) == n_ok
    assert abs((float(ls) - 0.75) - want) <= 1e-5 * abs(want)


def test_ce_all_rows_ignored(nat):
    M, V = 300, 1000
    labels = torch.full((M,), -100, dtype=torch.int64)
    labels[::3] = V
    ls = torch.full((1,), 2.5, dtype=torch.float32, device="cuda")
    nv = torch.full((1,), 7, dtype=torch.int32, device="cuda")
    d = torch.full((M, V), 1.0, dtype=torch.bfloat16, device="cuda")
    nat.ce_fwd_bwd(rnd(M, V, seed=30).cuda(), labels.cuda(), ls, nv, d, 1.0)
    assert float(ls) == 2.5 and int(nv) == 7
    assert float(d.float().abs().sum()) == 0.0


# ------------------------------------------------------------------------------------------------ embed_bwd
def _embed_ref(table, ids, dout):
    """token order, one bf16 rounding per add: equals one round-to-nearest of each exact pairwise sum (two bf16 values
    add exactly in fp32 when their exponents differ by at most 16; otherwise both forms return the larger one)"""
    acc = table.clone()
    V = acc.shape[0]
    for t, i in enumerate(ids.tolist()):
        if 0 <= i < V:
            acc[i] = (acc[i].float() + dout[t].float()).bfloat16()
    return acc


def _embed_ids(kind, n, g):
    if kind == "vocab8":                 # ids repeat across many warps
        return torch.randint(0, 8, (n,), generator=g), 8
    if kind == "same":
        return torch.full((n,), 5, dtype=torch.int64), 8
    if kind == "distinct":
        return torch.randperm(n, generator=g), n + 3
    if kind == "stride50":               # every repeat of an id lies 50 tokens back: the owner scan must reach it
        return torch.arange(n) % 50, 50
    if kind == "invalid":                # -100 and ids >= vocab leave the table untouched
        ids = torch.randint(0, 8, (n,), generator=g)
        ids[torch.rand(n, generator=g) < 0.3] = -100
        ids[torch.rand(n, generator=g) < 0.2] = 8
        ids[torch.rand(n, generator=g) < 0.1] = 1 << 40
        return ids, 8
    raise ValueError(kind)


@pytest.mark.parametrize("kind", ["vocab8", "same", "distinct", "stride50", "invalid"])
@pytest.mark.parametrize("H", [64, 896])
@pytest.mark.parametrize("n_tok", [1, 31, 32, 33, 1000, 4100])
def test_embed_bwd_token_order(nat, n_tok, H, kind):
    g = torch.Generator().manual_seed(31)
    ids, V = _embed_ids(kind, n_tok, g)
    dout = rnd(n_tok, H, seed=32)
    table = rnd(V, H, seed=33)
    want = _embed_ref(table, ids, dout)
    for _ in range(2):
        dt = table.cuda()
        nat.embed_bwd(ids.cuda(), dout.cuda(), dt)
        assert torch.equal(dt.cpu(), want)


# ------------------------------------------------------------------------------------------------ other reductions
@pytest.mark.parametrize("impl", ["mma", "wgmma"])
@pytest.mark.parametrize("B,S,n_h,n_kv,d", [(2, 130, 4, 2, 128), (1, 1024, 8, 2, 64)])
def test_attn_bwd_run_to_run(nat, monkeypatch, B, S, n_h, n_kv, d, impl):
    monkeypatch.setenv("TL_ATTN_BWD", impl)
    q, k, v = rnd(B, S, n_h, d, seed=34, std=0.7), rnd(B, n_kv, S, d, seed=35, std=0.7), rnd(B, n_kv, S, d, seed=36)
    do = rnd(B, S, n_h * d, seed=37).cuda()
    kc, vc, qd = k.cuda(), v.cuda(), q.cuda()
    out = torch.empty(B, S, n_h * d, dtype=torch.bfloat16, device="cuda")
    lse = torch.empty(B, n_h, S, dtype=torch.float32, device="cuda")
    nat.attn_prefill_fwd(qd, kc, vc, out, lse, B, S, 0, n_h, n_kv, d, d ** -0.5)
    res = []
    for _ in range(2):
        dq = torch.empty(B, S, n_h, d, dtype=torch.bfloat16, device="cuda")
        dk = torch.zeros(B, n_h, S, d, dtype=torch.bfloat16, device="cuda")
        dv = torch.zeros_like(dk)
        ws = torch.empty(nat.attn_bwd_ws(B, S, n_h), dtype=torch.uint8, device="cuda")
        nat.attn_bwd(qd, kc, vc, out, do, lse, dq, dk, dv, ws, B, S, n_h, n_kv, d, d ** -0.5)
        res.append((dq.cpu(), dk.cpu(), dv.cpu()))
    for a, b in zip(*res):
        assert torch.equal(a, b)
    assert float(res[0][0].float().abs().sum()) > 0


@pytest.mark.parametrize("M,N,K", [(100, 896, 4864), (9, 4608, 3584)])
def test_gemm_splitk_run_to_run(nat, M, N, K):
    a, w = rnd(M, K, seed=38).cuda(), rnd(N, K, seed=39, std=0.05).cuda()
    b, r = rnd(N, seed=40, std=0.5).cuda(), rnd(M, N, seed=41).cuda()
    ws = torch.empty(nat.gemm_splitk_ws(M, N), dtype=torch.uint8, device="cuda")
    for kw in ({"flags": nat.EPI_OUT_F32}, {"bias": b, "residual": r}):
        c1 = nat.gemm(a, w, ws=ws, **kw).cpu()
        c2 = nat.gemm(a, w, ws=ws, **kw).cpu()
        assert torch.equal(c1, c2), kw.keys()


def test_gemm_weight_gradient_accumulate_run_to_run(nat):
    """dW (+)= dy^T x with both operands MN-major and EPI_ACCUM, the lm_head / weight-gradient form"""
    M, N, K = 2048, 512, 2100
    dy, x = rnd(K, M, seed=42).cuda(), rnd(K, N, seed=43).cuda()
    c0 = rnd(M, N, seed=44).cuda()
    res = []
    for _ in range(2):
        c = c0.clone()
        nat.gemm(dy, x, out=c, flags=nat.A_MN_MAJOR | nat.B_MN_MAJOR | nat.EPI_ACCUM, M=M, K=K, N=N)
        res.append(c.cpu())
    assert torch.equal(res[0], res[1])
    assert O.rel_l2(res[0], c0.cpu().float() + dy.cpu().double().t() @ x.cpu().double()) <= TOL


# ------------------------------------------------------------------------------------------------ stream ordering
def _all_reductions(nat, src):
    """one call of each reduction on the current stream; inputs are copied from ``src`` on that stream first"""
    c = {k: v.clone() for k, v in src.items()}
    H, N, d = c["x"].shape[1], c["dy_b"].shape[1], c["qn"].shape[0]
    dx = torch.empty_like(c["x"])
    nat.rmsnorm_bwd(c["x"], c["w"], c["dy"], c["rstd"], dx, c["dw"])
    nat.colsum(c["dy_b"], c["db"])
    nat.qk_norm_bwd(c["pre"], c["dqkv"], c["qn"], c["kn"], c["gq"], c["gk"], 1e-6, 4, 2, d)
    dl = torch.empty_like(c["logits"])
    nat.ce_fwd_bwd(c["logits"], c["labels"], c["ls"], c["nv"], dl, 1e-3)
    nat.embed_bwd(c["ids"], c["dout"], c["table"])
    return {"dx": dx, "dw": c["dw"], "db": c["db"], "dqkv": c["dqkv"], "gq": c["gq"], "gk": c["gk"], "dl": dl,
            "ls": c["ls"], "nv": c["nv"], "table": c["table"]}


def test_reductions_follow_the_callers_stream(nat, sms):
    """The partial rows live in stream-ordered allocations on the caller's stream: inside torch.cuda.stream(side),
    with inputs produced on the side stream behind a delay, every result equals the default-stream call bit for bit."""
    rows, H, N, d, n_tok = 16 * sms + 1, 896, 1152, 128, 2000
    src = {"x": rnd(rows, H, seed=45, std=2.0), "w": rnd(H, seed=46), "dy": rnd(rows, H, seed=47),
           "dw": acc0(H, seed=48).float(), "dy_b": rnd(4097, N, seed=49), "db": acc0(N, seed=50).float(),
           "pre": rnd(n_tok, 8 * d, seed=51), "dqkv": rnd(n_tok, 8 * d, seed=52), "qn": rnd(d, seed=53),
           "kn": rnd(d, seed=54), "gq": acc0(d, seed=55).float(), "gk": acc0(d, seed=56).float(),
           "logits": rnd(2052, 1000, seed=57, std=2.0), "labels": torch.randint(0, 1000, (2052,)),
           "ls": torch.full((1,), 0.75), "nv": torch.zeros(1, dtype=torch.int32),
           "ids": torch.randint(0, 40, (n_tok,)), "dout": rnd(n_tok, H, seed=58), "table": rnd(40, H, seed=59)}
    src["rstd"] = torch.rsqrt(src["x"].float().pow(2).mean(-1) + 1e-6)
    src = {k: v.cuda() for k, v in src.items()}
    ref = _all_reductions(nat, src)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        torch.cuda._sleep(20_000_000)          # the side stream's inputs become ready well after the launches are issued
        got = _all_reductions(nat, src)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for k in ref:
        assert torch.equal(got[k], ref[k]), k
