"""Qwen3-MoE on the H100: the routing kernel and its grouped-GEMM plan, the grouped wgmma GEMM against tl_gemm_bf16, the
expert GEMV against float64, and tiny MoE models end to end against the MoE oracle (tests/moe_oracle.py).

Model-level criteria follow tests/test_model_gpu.py, with one addition: a token whose k-th and (k+1)-th router logits are
closer than the bf16 noise of two implementations may pick a different expert in each, which moves that position's
output by a whole expert's share.  So the accuracy / agreement bounds are applied to the positions' median error, and
at least 90 % of the positions must meet the agreement bound on their own."""
import pytest
import torch
import torch.nn.functional as F

from oracle import shard_oracle as O
from tensorlink_b200 import native as nat
from tensorlink_b200.ml import configs as C
from tensorlink_b200.ml.weights import init_state_dict, synthetic_tokens
from tests.moe_oracle import MoeOracleModel

pytestmark = pytest.mark.gpu
CASES = [C.TINY_QWEN3_MOE, C.TINY_QWEN3_MOE_UNNORM]
MARGIN = 0.05
dev = "cuda"


def _route(logits, k, norm, plan=True):
    N, E = logits.shape
    ids = torch.empty(N, k, dtype=torch.int32, device=dev)
    wts = torch.empty(N, k, dtype=torch.float32, device=dev)
    T = nat.moe_max_tiles(N, E, k)
    i32 = dict(dtype=torch.int32, device=dev)
    p = (torch.empty(E, **i32), torch.empty(E + 1, **i32), torch.empty(N * k, **i32), torch.empty(T, 2, **i32)) if plan else None
    nat.moe_route(logits, k, norm, ids, wts, p)
    torch.cuda.synchronize()
    return ids, wts, p


def _distinct_logits(N, E, seed):
    """bf16 logits with no two equal values in a row (no tie anywhere, so none at the k-th place)."""
    g = torch.Generator().manual_seed(seed)
    perm = torch.stack([torch.randperm(E, generator=g) for _ in range(N)])
    return ((perm.float() - E / 2) / 16).to(torch.bfloat16)


def _check_plan(ids, p, N, E, k):
    counts, offsets, row_of, tiles = (t.cpu() for t in p)
    ids = ids.cpu().long()
    assert torch.equal(counts.long(), torch.bincount(ids.flatten(), minlength=E))
    seg = (counts + 127) // 128 * 128
    assert torch.equal(offsets.long(), torch.cat([torch.zeros(1, dtype=torch.long), seg.cumsum(0)]))
    rows = row_of.view(N, k).long()
    for e in range(E):
        tok = (ids == e).nonzero()
        r = rows[ids == e]
        want = offsets[e] + torch.arange(len(tok))
        assert torch.equal(r, want.long()), e                                  # ascending token order, packed from the start
    for t in range(tiles.shape[0]):
        r0 = 128 * t
        if r0 < offsets[E]:
            e = int(torch.searchsorted(offsets[1:], torch.tensor(r0), right=True))
            assert tiles[t, 0] == e and tiles[t, 1] == min(128, int(counts[e]) - (r0 - int(offsets[e]))), t
        else:
            assert tiles[t, 0] == -1, t


@pytest.mark.parametrize("N,E,k", [(1, 32, 4), (7, 128, 8), (200, 128, 8), (1500, 256, 16), (33, 16, 16)])
@pytest.mark.parametrize("norm", [True, False])
def test_route_matches_topk_and_plan_is_consistent(N, E, k, norm):
    logits = _distinct_logits(N, E, N * E + k).to(dev)
    ids, wts, p = _route(logits, k, norm)
    pf = F.softmax(logits.float().cpu(), dim=-1)
    top, ref = torch.topk(pf, k, dim=-1)
    ref_sorted, order = ref.sort(dim=-1)
    assert torch.equal(ids.cpu().long(), ref_sorted)
    # float64 formula; the kernel's softmax sums its E terms in another order than torch, so the bound is 8 fp32 ulps
    p64 = F.softmax(logits.double().cpu(), dim=-1)
    top = torch.gather(p64, 1, ref)
    w = top / top.sum(-1, keepdim=True) if norm else top
    w = torch.gather(w, 1, order)
    assert bool(((wts.cpu().double() - w).abs() <= 8 * 2.0 ** -24 * w).all())
    _check_plan(ids, p, N, E, k)


def test_route_tie_picks_lower_index_and_skewed_plans():
    E, k = 64, 4
    logits = torch.zeros(3, E, dtype=torch.bfloat16)
    logits[0, [5, 9, 40, 41, 42]] = 1.0                                      # five-way tie for four places
    logits[1, [63, 0]] = 2.0
    logits[1, [10, 20, 30]] = 1.0
    ids, _, _ = _route(logits.to(dev), k, True, plan=False)
    assert ids[0].tolist() == [5, 9, 40, 41]
    assert ids[1].tolist() == [0, 10, 20, 63]
    assert ids[2].tolist() == [0, 1, 2, 3]                                   # all equal: the lowest indices
    for N in (1, 129, 1000):                                                  # every token on the same experts
        ids, _, p = _route(torch.zeros(N, E, dtype=torch.bfloat16, device=dev), k, True)
        _check_plan(ids, p, N, E, k)
    lg = torch.randn(300, E).bfloat16()
    lg[:, :6] += 20                                                           # most experts empty
    ids, _, p = _route(lg.to(dev), k, False)
    _check_plan(ids, p, 300, E, k)


@pytest.mark.parametrize("N,E,k,H,I", [(37, 32, 4, 512, 256), (300, 128, 8, 2048, 768)])
def test_grouped_gemm_equals_dense_gemm_per_expert(N, E, k, H, I):
    g = torch.Generator(device=dev).manual_seed(N)
    h = torch.randn(N, H, device=dev, generator=g).bfloat16()
    wgu = (torch.randn(E, 2 * I, H, device=dev, generator=g) * 0.02).bfloat16()
    wd = (torch.randn(E, H, I, device=dev, generator=g) * 0.02).bfloat16()
    logits = torch.randn(N, E, device=dev, generator=g).bfloat16()
    ids, wts, (counts, offsets, row_of, tiles) = _route(logits, k, True)
    T = tiles.shape[0]
    hg = torch.full((T * 128, H), float("nan"), device=dev).bfloat16()
    nat.moe_gather(h, row_of, hg, k)
    act = torch.full((T * 128, I), float("nan"), device=dev).bfloat16()
    y = torch.full((T * 128, H), float("nan"), device=dev).bfloat16()
    nat.moe_gemm(hg, wgu, act, tiles, flags=nat.EPI_SWIGLU)
    nat.moe_gemm(act, wd, y, tiles)
    out = torch.empty_like(h)
    nat.moe_combine(y, row_of, wts, h, out)
    torch.cuda.synchronize()
    ids_c, off = ids.cpu().long(), offsets.cpu()
    acc = torch.zeros(N, H)
    for e in range(E):
        tok = (ids_c == e).any(1).nonzero().flatten()
        if len(tok) == 0:
            continue
        r0 = int(off[e])
        rows = slice(r0, r0 + len(tok))
        assert torch.equal(hg[rows].cpu(), h[tok.to(dev)].cpu())
        a_ref = nat.gemm(h[tok.to(dev)].contiguous(), wgu[e], flags=nat.EPI_SWIGLU)
        assert torch.equal(act[rows], a_ref), e
        y_ref = nat.gemm(act[rows].contiguous(), wd[e])
        assert torch.equal(y[rows], y_ref), e
    # rows past each segment's count stay unwritten
    for e in range(E):
        c = int(counts[e])
        pad = slice(int(off[e]) + c, int(off[e + 1]))
        assert bool(torch.isnan(y[pad].float()).all()) and bool(torch.isnan(act[pad].float()).all())
    # combine: ascending expert order, bf16 accumulation from +0, then the residual
    yc, wc = y.cpu().float(), wts.cpu()
    rc = row_of.cpu().view(N, k).long()
    for s in range(k):
        c = (yc[rc[:, s]] * wc[:, s:s + 1]).bfloat16().float()
        acc = (acc + c).bfloat16().float()
    assert torch.equal(out.cpu(), (h.cpu().float() + acc).bfloat16())


def _ints(shape, lo, hi, scale, g):
    return (torch.randint(lo, hi + 1, shape, device=dev, generator=g).float() * scale).bfloat16()


@pytest.mark.parametrize("M", [1, 2, 3, 8])
def test_expert_gemv_bit_exact_vs_gemv(M):
    """Exact-integer inputs: every fp32 dot product is exact whatever the summation order, so each rounding point shows.
    gate/up: each (row, pick) equals tl_gemv_bf16 (EPI_SWIGLU) on that expert's slice at the same row count, bit for bit.
    down: equals HF's combine applied on the CPU to tl_gemv_bf16 outputs of each picked expert's down slice."""
    E, k, H, I = 32, 4, 512, 256
    g = torch.Generator(device=dev).manual_seed(M)
    x = _ints((M, H), -8, 8, 2.0 ** -4, g)
    wgu = _ints((E, 2 * I, H), -8, 8, 2.0 ** -8, g)
    wd = _ints((E, H, I), -8, 8, 2.0 ** -8, g)
    ids, wts, _ = _route(torch.randn(M, E, device=dev, generator=g).bfloat16(), k, True, plan=False)
    act = torch.empty(M * k, I, device=dev).bfloat16()
    nat.moe_gemv(x, wgu, act, ids, flags=nat.EPI_SWIGLU)
    a_in = _ints((M * k, I), -8, 8, 2.0 ** -4, g)          # the down launch's input, exact too
    res = torch.randn(M, H, device=dev, generator=g).bfloat16()
    out = torch.empty(M, H, device=dev).bfloat16()
    nat.moe_gemv(a_in, wd, out, ids, wts=wts, residual=res, flags=nat.EPI_RESIDUAL)
    torch.cuda.synchronize()
    idc = ids.cpu().long()
    acc = torch.zeros(M, H)
    for r in range(M):
        for s in range(k):
            e = int(idc[r, s])
            ref = nat.gemv(x, wgu[e], flags=nat.EPI_SWIGLU)[r]
            assert torch.equal(act[r * k + s], ref), (r, s)
    for s in range(k):
        ys = torch.stack([nat.gemv(a_in.view(M, k, I)[:, s].contiguous(), wd[int(idc[r, s])])[r] for r in range(M)]).cpu()
        acc = (acc + (ys.float() * wts.cpu()[:, s:s + 1]).bfloat16().float()).bfloat16().float()
    want = (res.cpu().float() + acc).bfloat16()
    assert torch.equal(out.cpu().view(torch.int16), want.view(torch.int16))


def test_expert_gemv_negative_zero_contributions():
    """Every contribution -0 (y = +0 times a negative weight) on a -0 residual: HF's accumulator starts at +0 and
    +0 + -0 = +0, so the output is +0; an accumulator started at -0 would give -0."""
    E, k, H, I = 32, 4, 512, 256
    g = torch.Generator(device=dev).manual_seed(3)
    ids, _, _ = _route(torch.randn(2, E, device=dev, generator=g).bfloat16(), k, True, plan=False)
    wts = -torch.rand(2, k, device=dev, generator=g) - 0.1
    act = torch.randn(2 * k, I, device=dev, generator=g).bfloat16()
    wd = torch.zeros(E, H, I, device=dev).bfloat16()
    res = torch.full((2, H), -0.0, device=dev).bfloat16()
    out = torch.empty(2, H, device=dev).bfloat16()
    nat.moe_gemv(act, wd, out, ids, wts=wts, residual=res, flags=nat.EPI_RESIDUAL)
    assert bool((out.view(torch.int16) == 0).all())
    y = torch.zeros(2 * k, H, device=dev).bfloat16()                    # the grouped path's combine, same rule
    row_of = torch.arange(2 * k, dtype=torch.int32, device=dev)
    out2 = torch.empty(2, H, device=dev).bfloat16()
    nat.moe_combine(y, row_of, wts, res, out2)
    assert bool((out2.view(torch.int16) == 0).all())


@pytest.mark.parametrize("M", [1, 3, 8])
def test_expert_gemv_vs_float64(M):
    """Random inputs: within one bf16 rounding of the float64 dot products (the fp32 sums differ from float64)."""
    E, k, H, I = 32, 4, 512, 256
    g = torch.Generator(device=dev).manual_seed(M)
    x = torch.randn(M, H, device=dev, generator=g).bfloat16()
    wgu = (torch.randn(E, 2 * I, H, device=dev, generator=g) * 0.05).bfloat16()
    ids, _, _ = _route(torch.randn(M, E, device=dev, generator=g).bfloat16(), k, True, plan=False)
    act = torch.empty(M * k, I, device=dev).bfloat16()
    nat.moe_gemv(x, wgu, act, ids, flags=nat.EPI_SWIGLU)
    torch.cuda.synchronize()
    idc, xd, gu = ids.cpu().long(), x.cpu().double(), wgu.cpu().double()
    for r in range(M):
        for s in range(k):
            z = gu[idc[r, s]] @ xd[r]
            gt, up = z[0::2].bfloat16().float(), z[1::2].bfloat16().float()
            ref = (F.silu(gt).bfloat16().float() * up)
            got = act[r * k + s].cpu().float()
            assert bool(((got - ref).abs() <= ref.abs() * 2.0 ** -7 + 1e-6).all()), (r, s)


def make(cfg, **kw):
    from tensorlink_b200.ml import DistributedModel
    kw.setdefault("max_seq", 256)
    return DistributedModel(cfg, training=False, **kw)


def _positions_check(got, ref_bf16, ref_f32):
    """Returns the positions whose agreement is outside the bound (a router pick that differs at a near tie)."""
    S = got.shape[1]
    e_ref = torch.tensor([O.rel_l2(ref_bf16[:, s], ref_f32[:, s]) for s in range(S)])
    e_gpu = torch.tensor([O.rel_l2(got[:, s], ref_f32[:, s]) for s in range(S)])
    mutual = torch.tensor([O.rel_l2(got[:, s], ref_bf16[:, s]) for s in range(S)])
    assert e_gpu.median() <= 1.5 * e_ref.median(), (e_gpu.median(), e_ref.median())
    assert mutual.median() <= 2 * e_ref.median(), (mutual.median(), e_ref.median())
    assert (mutual <= 2 * e_ref).float().mean() >= 0.9, mutual / e_ref
    return mutual > 2 * e_ref


@pytest.mark.parametrize("cfg", CASES, ids=lambda c: c.name)
def test_prefill_logits_vs_oracle(cfg):
    sd = init_state_dict(cfg)
    ids = synthetic_tokens(cfg, 1, 64)
    got = make(cfg)(ids).logits.cpu().float()
    with torch.no_grad():
        ref = MoeOracleModel(cfg, sd, "sdpa_math").logits(ids).float()
        ref32 = MoeOracleModel(cfg, {k: v.float() for k, v in sd.items()}, "sdpa_math").logits(ids)
    _positions_check(got, ref, ref32)


def _check_ids(got, ref, margins, prompt_len):
    n = 0
    for b in range(got.shape[0]):
        for s in range(got.shape[1] - prompt_len):
            if margins[b, s] < MARGIN:
                break
            assert got[b, prompt_len + s] == ref[b, prompt_len + s], f"row {b} step {s}: margin {margins[b, s]:.3f}"
            n += 1
    return n


@pytest.mark.parametrize("cfg", CASES, ids=lambda c: c.name)
@pytest.mark.parametrize("B", [1, 3, 8, 32])
def test_greedy_decode_rows_vs_oracle_and_graph_equals_eager(cfg, B):
    sd = init_state_dict(cfg)
    ids = synthetic_tokens(cfg, B, 10, seed=B)
    dm = make(cfg, max_batch=B)
    got = dm.generate(ids, max_new_tokens=12).cpu()
    eager = dm.generate(ids, max_new_tokens=12, use_graph=False).cpu()
    again = dm.generate(ids, max_new_tokens=12).cpu()
    assert torch.equal(got, eager) and torch.equal(got, again)
    ref, margins = MoeOracleModel(cfg, sd, "sdpa_math").generate(ids, 12, return_margins=True)
    n = _check_ids(got, ref, margins, 10)
    # teacher-forced: each generated token is the oracle's argmax over the generated sequence wherever that margin is
    # resolvable, independent of earlier forks (tests/test_model_gpu.py)
    with torch.no_grad():
        lf = MoeOracleModel(cfg, sd, "sdpa_math").logits(got[:, :-1])[:, 9:].float()
    top2 = lf.topk(2, dim=-1).values
    safe = (top2[..., 0] - top2[..., 1]) >= MARGIN
    assert int(safe.sum()) >= 3, int(safe.sum())
    assert torch.equal(got[:, 10:][safe], lf.argmax(-1)[safe])
    print(f"{cfg.name} B={B}: {n} steps exact, {int(safe.sum())} teacher-forced")


def test_left_padded_row_equals_row_alone_and_sampling_reproducible():
    cfg = C.TINY_QWEN3_MOE
    dm = make(cfg, max_batch=2)
    a = synthetic_tokens(cfg, 1, 12, seed=1)
    b = synthetic_tokens(cfg, 1, 7, seed=2)
    ids = torch.cat([torch.cat([torch.zeros(1, 5, dtype=torch.long), b], 1), a])
    mask = torch.ones_like(ids)
    mask[0, :5] = 0
    both = dm.generate(ids, attention_mask=mask, max_new_tokens=10).cpu()
    alone = dm.generate(b, max_new_tokens=10).cpu()
    assert torch.equal(both[0, 5:], alone[0])
    kw = dict(max_new_tokens=12, do_sample=True, temperature=0.9, top_k=20, seed=7)
    assert torch.equal(dm.generate(a, **kw).cpu(), dm.generate(a, **kw).cpu())


def test_output_scores():
    cfg = C.TINY_QWEN3_MOE_UNNORM
    dm = make(cfg, max_batch=1)
    ids = synthetic_tokens(cfg, 1, 16, seed=5)
    plain = dm.generate(ids, max_new_tokens=6).cpu()
    out = dm.generate(ids, max_new_tokens=6, output_scores=True, return_dict_in_generate=True)
    assert len(out.scores) == 6 and torch.equal(out.sequences.cpu(), plain)
    for s, sc in enumerate(out.scores):
        assert int(sc.argmax(-1)) == int(plain[0, ids.shape[1] + s])


def _reliable(margins):
    bad = (margins[0] < MARGIN).nonzero()
    return int(bad[0]) if bad.numel() else margins[0].numel()


@pytest.mark.parametrize("cfg", CASES, ids=lambda c: c.name)
@pytest.mark.parametrize("K", [1, 2, 3, 10])
def test_prompt_lookup_vs_greedy(cfg, K):
    """As tests/test_prompt_lookup_gpu.py: a verify step is not bit-identical to decode steps (its attention and, above
    gemv_rows() rows, its Linears differ), so the tokens equal plain greedy decoding's and the oracle's up to the first
    step whose oracle margin is unresolvable; graph replay equals eager launches bit for bit."""
    sd = init_state_dict(cfg)
    ids = synthetic_tokens(cfg, 1, 8).repeat(1, 3)
    S, new = ids.shape[1], 32
    ref, margins = MoeOracleModel(cfg, sd, "sdpa_math").generate(ids, new, return_margins=True)
    dm = make(cfg, max_batch=1)
    plain = dm.generate(ids, max_new_tokens=new).cpu()
    got = dm.generate(ids, max_new_tokens=new, prompt_lookup_num_tokens=K).cpu()
    eager = dm.generate(ids, max_new_tokens=new, prompt_lookup_num_tokens=K, use_graph=False).cpu()
    assert torch.equal(got, eager)
    n_ok = _reliable(margins)
    _check_ids(got, ref, margins, S)
    assert torch.equal(got[:, S:S + n_ok], plain[:, S:S + n_ok])


def test_assisted_vs_greedy():
    cfg = C.TINY_QWEN3_MOE
    sd = init_state_dict(cfg)
    ids = synthetic_tokens(cfg, 1, 12, seed=9)
    ref, margins = MoeOracleModel(cfg, sd, "sdpa_math").generate(ids, 24, return_margins=True)
    dm = make(cfg, max_batch=1)
    helper = make(cfg.scaled(n_layers=1, name="tiny-qwen3-moe-1l"), max_batch=1)
    plain = dm.generate(ids, max_new_tokens=24).cpu()
    got = dm.generate(ids, max_new_tokens=24, assistant_model=helper, num_assistant_tokens=3).cpu()
    n_ok = _reliable(margins)
    _check_ids(got, ref, margins, 12)
    assert torch.equal(got[:, 12:12 + n_ok], plain[:, 12:12 + n_ok])


def test_verify_rows_route_like_decode_steps():
    """Row by row, a 3-row verify step (the expert GEMV path) against three 1-row decode steps from the same cache: the
    last layer's router logits agree to bf16 noise, and its picks are the same wherever the k-th / (k+1)-th logit gap
    is above that noise."""
    cfg = C.TINY_QWEN3_MOE
    dm = make(cfg, max_batch=1)
    st = dm.stage
    cg = st.slots[0]
    ids = synthetic_tokens(cfg, 1, 20, seed=11)
    S = 16
    hs = st.embed(ids.to(dev))[0]
    cg.prefill(hs[:S].unsqueeze(0).contiguous())
    dec_logits, dec_ids, dec_out = [], [], []
    for i in range(S, S + 3):
        x = hs[i:i + 1].clone()
        cg.decode_step_inplace(x)
        dec_out.append(x[0].clone())
        dec_logits.append(cg.dbufs.moe.logits[0].float().clone())
        dec_ids.append(cg.dbufs.moe.ids[0].clone())
    cg.reset_cache(S)
    xv = hs[S:S + 3].clone()
    cg.verify_step_inplace(xv)
    torch.cuda.synchronize()
    for r in range(3):
        lv, ld = cg.vbufs.moe.logits[r].float(), dec_logits[r]
        assert float((lv - ld).abs().max()) <= 0.05 * float(ld.abs().max()), r
        srt = ld.sort(descending=True).values
        if float(srt[cfg.top_k - 1] - srt[cfg.top_k]) > 4 * float((lv - ld).abs().max()) + 1e-3:
            assert torch.equal(cg.vbufs.moe.ids[r], dec_ids[r]), r
        assert O.rel_l2(xv[r], dec_out[r]) < 0.02, r


def test_full_width_one_layer_vs_oracle():
    """One layer of Qwen3-30B-A3B width (E 128, k 8, I_e 768) with the full-vocabulary lm_head: prefill 192 and
    four decode steps against the oracle."""
    cfg = C.QWEN3_30B_A3B.scaled(n_layers=1, name="qwen3-30b-a3b-1layer")
    sd = init_state_dict(cfg)
    ids = synthetic_tokens(cfg, 1, 192)
    dm = make(cfg, max_seq=256)
    got = dm(ids).logits.cpu().float()
    with torch.no_grad():
        ref = MoeOracleModel(cfg, sd, "sdpa_math").logits(ids).float()
        ref32 = MoeOracleModel(cfg, {k: v.float() for k, v in sd.items()}, "sdpa_math").logits(ids)
    flipped = _positions_check(got, ref, ref32)
    top2 = ref[0].topk(2, dim=-1).values
    safe = (top2[:, 0] - top2[:, 1]) >= MARGIN
    assert int(safe.sum()) >= 50, int(safe.sum())
    # at a resolvable margin the argmax agrees, except at positions whose output moved by a different router pick
    differ = got[0].argmax(-1) != ref[0].argmax(-1)
    assert not bool((differ & safe & ~flipped).any()), (differ & safe).nonzero().flatten()
    gen = dm.generate(ids, max_new_tokens=4).cpu()
    want, margins = MoeOracleModel(cfg, sd, "sdpa_math").generate(ids, 4, return_margins=True)
    _check_ids(gen, want, margins, 192)


def test_training_and_optimizer_raise():
    with pytest.raises(NotImplementedError):
        make(C.TINY_QWEN3_MOE).create_optimizer()
