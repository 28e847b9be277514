"""Sampling with drafts on the GPU: ``generate(do_sample=True)`` with ``assistant_model`` (speculative sampling,
csrc/sample.cu ``tl_spec_accept``) and with ``prompt_lookup_num_tokens`` (one draw per verify row, the agreeing prefix).

  1. the kernel draw by draw: crafted p / q rows, replayed on the CPU with the sampler's float64 model
     (tests/rowwise_cases.py ``sample_row_model``, ``philox_u``).  A decision or a draw may differ from the replay only
     where u lies inside the weights' error band of p/q or of a CDF boundary; those cases are counted.  The counter
     advance, the exclusion of the rejected draft and ``pl_accept``'s prefix are exact;
  2. the kernel's full law: drafts drawn by ``tl_sample`` from fixed q rows, then ``tl_spec_accept``, 20,000 times,
     against prod_{i<n} min(p_i, q_i)(d_i) * (p_n - q_n)+(t), or * p_K(t) when every draft is kept (chi-square);
  3. the stage round by round: every eager ``verify_round`` replayed from the rows its kernels read; graph == eager;
     seeds reproduce and differ; an identical assistant keeps almost every draft;
  4. generate's output distribution over seeds against the model's own teacher-forced warped distribution, EOS and
     max_new_tokens boundaries, the streamer;
  5. mismatched vocabularies, and a Qwen2.5-7B model with a Qwen2.5-0.5B assistant at full size.
"""
import functools
import itertools

import numpy as np
import pytest
import torch

from tensorlink_b200.ml import configs as C
from tensorlink_b200.ml.module import apply_eos
from tensorlink_b200.ml.stage import (CTR_ACCEPT, CTR_DRAFTS, STREAM_ACCEPT, STREAM_DRAFTS, STREAM_PL_ROWS,
                                      stream_seed)
from tensorlink_b200.ml.weights import synthetic_tokens
from tests.rowwise_cases import RowModel, check_draws, philox_u, sample_row_model

pytestmark = pytest.mark.gpu
DRAW_ROW = 16                   # tl_spec_accept's Philox row of the final draw
CASES = [C.TINY_QWEN2, C.TINY_QWEN2_D128, C.TINY_QWEN3]


@pytest.fixture(scope="module")
def nat():
    from tensorlink_b200 import native
    native.require_device()
    return native


def _chi2_ok(counts, exp):
    big = exp >= 5
    chi2 = float((((counts - exp) ** 2) / np.maximum(exp, 1e-12))[big].sum())
    dof = int(big.sum()) - 1
    return chi2 < dof + 6 * (2 * dof) ** 0.5 + 10, (chi2, dof)       # ~6 sigma, as tests/test_sampling_gpu.py


# ------------------------------------------------------------------------------------------ CPU replay
def _prob(rm: RowModel, d):
    """(p(d), its error bound) of a row model: weight / Z_kept"""
    if not 0 <= d < len(rm.w):
        return 0.0, 0.0
    Z = rm.Zk
    return rm.w[d] / Z, (rm.err[d] + rm.w[d] * rm.err.sum() / Z) / Z


def _residual_model(pm: RowModel, qm: RowModel, d):
    """(p - q)+ over the target's ids, the rejected draft d excluded, with its error bound per id"""
    Vp, Vq = len(pm.w), len(qm.w)
    m = min(Vp, Vq)
    wq, eq = np.zeros(Vp), np.zeros(Vp)
    wq[:m], eq[:m] = qm.w[:m], qm.err[:m]
    Zp, Zq = pm.Zk, qm.Zk
    raw = pm.w / Zp - wq / Zq
    er = pm.err / Zp + pm.w * pm.err.sum() / Zp ** 2 + eq / Zq + wq * qm.err.sum() / Zq ** 2
    r = np.maximum(raw, 0.0)
    if 0 <= d < Vp:
        r[d] = 0.0
    er = np.where((raw > -er) & (r > 0), er, 0.0)
    return RowModel(r > 0, r, er, np.cumsum(r), float(r.sum()), False, True)


def spec_replay(name, pm, qm, drafts, u_acc, u_draw, got, errors):
    """Check the kernel's ids ``got`` against the replay of tl_spec_accept; returns (n, in-band cases)."""
    nc = len(drafts)
    n = next((i for i in range(nc) if got[i] != drafts[i]), nc)          # the kernel's first rejection
    band = 0
    for i in range(min(n + 1, nc)):
        p, ep = _prob(pm[i], drafts[i])
        q, eq = _prob(qm[i], drafts[i])
        b = u_acc[i] * eq + ep
        near = b > 0 and abs(u_acc[i] * q - p) <= b
        band += near
        if (u_acc[i] * q < p) != (i < n) and not near:
            errors.append(f"{name}: draft {i} ({drafts[i]}) {'kept' if i < n else 'rejected'} with u={u_acc[i]:.6f} "
                          f"q={q:.6g} p={p:.6g}")
    tok = got[n]
    if n < nc:
        if tok == drafts[n]:
            errors.append(f"{name}: the rejected draft {tok} was drawn")
        rm = _residual_model(pm[n], qm[n], drafts[n])
        if rm.Zk <= 4 * rm.err.sum():
            return n, band + 1                       # the residual rounds to ~0: the kernel may fall back to p_n
    else:
        rm = pm[n]
    if not 0 <= tok < len(pm[n].w):
        errors.append(f"{name}: token {tok} outside the target's vocabulary")
        return n, band
    return n, band + check_draws(f"{name} draw", [tok], rm, np.array([u_draw]), errors)


def _row_models(rows, T, top_k, top_p):
    return [sample_row_model(r, T, top_k, top_p) for r in rows]


# ------------------------------------------------------------------------------------------ 1. the kernel, draw by draw
KERNEL_CASES = [  # name, K, V_p, V_q, temperature, top_k, top_p, ties at the top
    ("V8.K1", 1, 8, 8, 1.0, 0, 1.0, False),
    ("V8.K2.k3", 2, 8, 8, 1.0, 3, 1.0, False),
    ("V1000.K4.p", 4, 1000, 1000, 0.7, 0, 0.8, True),
    ("V1000.K15.k40", 15, 1000, 1000, 1.0, 40, 1.0, False),
    ("V152064_151936.K4.k50", 4, 152064, 151936, 1.0, 50, 1.0, False),
    ("V151936_152064.K15.k50p", 15, 151936, 152064, 1.0, 50, 0.9, False),
]


def _crafted_rows(K, Vp, Vq, ties, seed):
    g = torch.Generator().manual_seed(seed)
    V = max(Vp, Vq)
    x = torch.randn(K + 1, V, generator=g, dtype=torch.float64) * 2.0
    y = x[:K] + torch.randn(K, V, generator=g, dtype=torch.float64) * 0.8      # p > q on some ids, p < q on others
    if ties:                                          # a group of equal logits at the top, cut by top-p
        x = torch.minimum(x, torch.tensor(3.0))
        x[:, :10] = 3.0
        y = torch.minimum(y, torch.tensor(3.0))
        y[:, 5:15] = 3.0
    return x[:, :Vp].to(torch.bfloat16).contiguous(), y[:, :Vq].to(torch.bfloat16).contiguous()


def _pick_drafts(rng, pm, qm, K, Vp, Vq):
    """per draft: from q (most), p's top, an id p drops, an id the target lacks, or any id"""
    out = []
    for i in range(K):
        kind = rng.random()
        if kind < 0.5:
            w = qm[i].w / qm[i].w.sum()
            out.append(int(rng.choice(len(w), p=w)))
        elif kind < 0.65:
            out.append(int(np.argmax(pm[i].w)))
        elif kind < 0.8 and (pm[i].w == 0).any():
            out.append(int(rng.choice(np.nonzero(pm[i].w == 0)[0])))
        elif kind < 0.9 and Vq > Vp:
            out.append(int(rng.integers(Vp, Vq)))
        else:
            out.append(int(rng.integers(0, max(Vp, Vq))))
    return out


@pytest.mark.parametrize("case", KERNEL_CASES, ids=lambda c: c[0])
def test_spec_accept_draw_by_draw(nat, case):
    name, K, Vp, Vq, T, top_k, top_p, ties = case
    P, Q = _crafted_rows(K, Vp, Vq, ties, seed=K * 7 + Vp)
    pm, qm = _row_models(P, T, top_k, top_p), _row_models(Q, T, top_k, top_p)
    assert all(m.pinned for m in pm + qm), "a top-p boundary lies inside its error band (case not pinned)"
    seed = 0x1234_5678_9ABC_DEF0 + K
    trials = 200 if Vp <= 1000 else 24
    rng = np.random.default_rng(K + Vp)
    dev = "cuda"
    Pd, Qd = P.to(dev), Q.to(dev)
    ws = torch.empty(nat.spec_accept_ws(K), dtype=torch.uint8, device=dev)
    L = 64
    runs = []
    for t in range(trials):
        drafts = _pick_drafts(rng, pm, qm, K, Vp, Vq)
        nc = K if t % 4 else int(rng.integers(0, K + 1))              # some steps with fewer candidates
        ctr0 = 1000 * t + 7
        in_ids = torch.tensor([5] + drafts, dtype=torch.int64, device=dev)
        n_cand = torch.tensor([nc], dtype=torch.int32, device=dev)
        ctr = torch.tensor([ctr0], dtype=torch.int32, device=dev)
        ids = torch.full((K + 1,), -7, dtype=torch.int64, device=dev)
        nat.spec_accept(Pd, Qd, in_ids, n_cand, ctr, ids, ws, T, top_k, top_p, seed)
        # pl_accept after it: the kept drafts and the drawn token join a fresh history and the output log
        log = torch.zeros(L, dtype=torch.int32, device=dev)
        length = torch.tensor([3], dtype=torch.int32, device=dev)
        params = nat.pl_params(2, L, []).to(dev)
        out_log = torch.full((32,), -9, dtype=torch.int64, device=dev)
        count, pos, kvl = (torch.tensor([v], dtype=torch.int32, device=dev) for v in (0, 10, 10))
        nat.pl_accept(ids, in_ids, n_cand, log, length, None, Vp, params, out_log, count, pos, kvl, K)
        runs.append((drafts[:nc], ctr0, ctr, ids, out_log, count))
    errors, band, n_hist = [], 0, np.zeros(K + 1, np.int64)
    for t, (drafts, ctr0, ctr, ids, out_log, count) in enumerate(runs):
        got = ids.cpu().tolist()
        assert int(ctr.item()) == ctr0 + 1, "the counter advances by one per call"
        u_acc = [float(philox_u(seed, i, [ctr0])[0]) for i in range(len(drafts))]
        u_draw = float(philox_u(seed, DRAW_ROW, [ctr0])[0])
        n, b = spec_replay(f"{name} trial {t}", pm, qm, drafts, u_acc, u_draw, got, errors)
        band += b
        n_hist[n] += 1
        assert got[n + 1:] == [-7] * (K - n), "ids after the drawn token are not written"
        assert int(count.item()) == n + 1 and out_log[:n + 1].cpu().tolist() == got[:n + 1]
    print(f"{name}: {trials} steps, first rejection histogram {n_hist.tolist()}, {band} in-band cases")
    assert not errors, "\n".join(errors[:10])
    assert band <= max(2, trials // 20)


# ------------------------------------------------------------------------------------------ 2. the kernel, the full law
@pytest.mark.parametrize("K,top_k,top_p", [(2, 4, 1.0), (3, 0, 0.9)])
def test_spec_accept_law(nat, K, top_k, top_p):
    V, N, T = 6, 20000, 1.0
    g = torch.Generator().manual_seed(11 + K)
    P = (torch.randn(K + 1, V, generator=g) * 1.2).bfloat16()
    Q = (P[:K].float() + torch.randn(K, V, generator=g) * 0.9).bfloat16()
    pm, qm = _row_models(P, T, top_k, top_p), _row_models(Q, T, top_k, top_p)
    assert all(m.pinned for m in pm + qm)
    p = [m.w / m.Zk for m in pm]
    q = [m.w / m.Zk for m in qm]
    dev = "cuda"
    Pd, Qd = P.to(dev), Q.to(dev)
    ws_q = torch.empty(nat.sample_ws(K), dtype=torch.uint8, device=dev)
    ws = torch.empty(nat.spec_accept_ws(K), dtype=torch.uint8, device=dev)
    ctr_q = torch.zeros(K, dtype=torch.int32, device=dev)
    ctr = torch.zeros(1, dtype=torch.int32, device=dev)
    in_ids = torch.zeros(K + 1, dtype=torch.int64, device=dev)
    n_cand = torch.tensor([K], dtype=torch.int32, device=dev)
    rec = torch.zeros(N, 2 * K + 1, dtype=torch.int64, device=dev)
    for j in range(N):
        nat.sample(Qd, in_ids[1:], ctr_q, ws_q, T, top_k, top_p, 77)
        nat.spec_accept(Pd, Qd, in_ids, n_cand, ctr, rec[j, K:], ws, T, top_k, top_p, 78)
        rec[j, :K].copy_(in_ids[1:])
    rec = rec.cpu().numpy()
    assert int(ctr.item()) == N and (ctr_q.cpu() == N).all()
    # the exact law of the emitted tuple (d_0..d_{n-1}, t)
    law = {}
    for n in range(K + 1):
        for pre in itertools.product(range(V), repeat=n):
            w = float(np.prod([min(p[i][d], q[i][d]) for i, d in enumerate(pre)]))
            last = np.maximum(p[n] - q[n], 0.0) if n < K else p[K]
            for t in range(V):
                if w * last[t] > 0:
                    law[pre + (t,)] = law.get(pre + (t,), 0.0) + w * last[t]
    assert abs(sum(law.values()) - 1.0) < 1e-9
    counts = {}
    for row in rec:
        drafts, got = row[:K].tolist(), row[K:].tolist()
        n = next((i for i in range(K) if got[i] != drafts[i]), K)
        key = tuple(got[:n + 1])
        counts[key] = counts.get(key, 0) + 1
    outside = sum(c for k, c in counts.items() if k not in law)
    assert outside == 0, f"{outside} outcomes of probability 0"
    keys = sorted(law)
    ok, stat = _chi2_ok(np.array([counts.get(k, 0) for k in keys], float), np.array([law[k] for k in keys]) * N)
    assert ok, stat
    first = np.bincount(rec[:, K], minlength=V).astype(float)          # the first emitted token follows p_0
    ok0, stat0 = _chi2_ok(first, p[0] * N)
    print(f"K={K}: {len(counts)} outcomes of {len(law)}, chi2 {stat}, first token chi2 {stat0}")
    assert ok0, stat0


# ------------------------------------------------------------------------------------------ models
def _make(cfg, seed=1234, **kw):
    from tensorlink_b200.ml import DistributedModel
    kw.setdefault("max_seq", 256)
    kw.setdefault("max_batch", 1)
    return DistributedModel(cfg, training=False, seed=seed, **kw)


@functools.lru_cache(maxsize=None)
def _target(cfg):
    return _make(cfg)


@functools.lru_cache(maxsize=None)
def _assistant(cfg, kind):
    if kind == "lookup":
        return None
    return _make(cfg.scaled(n_layers=2) if kind == "two_layers" else cfg, seed=99 if kind == "other_seed" else 1234)


def _prompt(cfg, kind):
    ids = synthetic_tokens(cfg, 1, 12)
    if kind == "lookup":                              # self-repeating, so the n-gram lookup finds drafts
        ids = ids[:, :5].repeat(1, 3)
    return ids


def _sampling(seed, top_k=4, temperature=1.0, top_p=1.0):
    return {"temperature": temperature, "top_k": top_k, "top_p": top_p, "seed": seed}


# ------------------------------------------------------------------------------------------ 3. the stage, round by round
def _begin(dm, draft, ids, K, sampling, new):
    st = dm.stage
    st.set_sampling(sampling)
    st.sample_ctr.zero_()
    st.set_logits_processors(None)
    ids = ids.cuda()
    x = st.prefill(st.embed(ids), 0, 0)
    first = st.ids_dec[0][:1]
    st.head_argmax(x[:, -1, :].contiguous(), first, 0)
    if draft is not None:
        draft.stage.prefill(draft.stage.embed(ids), 0, 0)
    st.prompt_lookup_begin(torch.cat([ids, first.view(1, 1)], dim=1), K, 2, ids.shape[1] + new, [],
                           assistant=None if draft is None else draft.stage)


def replay_round(name, st, ast, s, ctr0, drafts, emitted, errors, overlap=None):
    """One eager round against its CPU replay; returns (kept drafts, in-band cases).  ``overlap`` (a list) collects
    sum_t min(p_i, q_i)(t), the probability that draft i is kept, for every assistant row."""
    K = st.pl_K
    warp = (s["temperature"], s["top_k"], s["top_p"])
    pm = _row_models(st.pl["logits"][:K + 1].cpu(), *warp)
    ctr1 = st.pl["ctr"].cpu().numpy().astype(np.int64)
    got = st.pl["ids"][:K + 1].cpu().tolist()
    band = 0
    if ast is None:
        for i in range(K + 1):                         # every row drawn from its own warped distribution
            u = philox_u(stream_seed(s["seed"], STREAM_PL_ROWS), i, [ctr0[i]])
            band += check_draws(f"{name} row {i}", [got[i]], pm[i], u, errors)
        assert (ctr1[:K + 1] == ctr0[:K + 1] + 1).all() and (ctr1[K + 1:] == ctr0[K + 1:]).all()
        n = next((i for i in range(len(drafts)) if got[i] != drafts[i]), len(drafts))
    else:
        qm = _row_models(ast.asst["q"][:K].cpu(), *warp)
        if overlap is not None and len(qm[0].w) == len(pm[0].w):
            overlap += [float(np.minimum(pm[i].w / pm[i].Zk, qm[i].w / qm[i].Zk).sum()) for i in range(K)]
        for i in range(K):                             # draft i drawn from the assistant's row i
            u = philox_u(stream_seed(s["seed"], STREAM_DRAFTS), 0, [ctr0[CTR_DRAFTS] + i])
            band += check_draws(f"{name} draft {i}", [drafts[i]], qm[i], u, errors)
        c = ctr0[CTR_ACCEPT]
        u_acc = [float(philox_u(stream_seed(s["seed"], STREAM_ACCEPT), i, [c])[0]) for i in range(K)]
        u_draw = float(philox_u(stream_seed(s["seed"], STREAM_ACCEPT), DRAW_ROW, [c])[0])
        n, b = spec_replay(name, pm, qm, drafts, u_acc, u_draw, got, errors)
        band += b
        assert ctr1[CTR_DRAFTS] == ctr0[CTR_DRAFTS] + K and ctr1[CTR_ACCEPT] == c + 1
    assert emitted == got[:n + 1], (name, emitted, got, drafts)
    return n, band


@pytest.mark.parametrize("cfg", CASES, ids=lambda c: c.name)
@pytest.mark.parametrize("kind", ["same", "other_seed", "two_layers", "lookup"])
@pytest.mark.parametrize("K", [1, 4])
def test_rounds_replayed(cfg, kind, K):
    dm, draft = _target(cfg), _assistant(cfg, kind)
    s = _sampling(4242 + K)
    rounds, new = 8, 8 * (K + 1) + 4
    _begin(dm, draft, _prompt(cfg, kind), K, s, new)
    st = dm.stage
    errors, band, kept, n_drafts, overlap = [], 0, 0, 0, []
    for r in range(rounds):
        ctr0 = st.pl["ctr"].cpu().numpy().astype(np.int64)
        drafts, emitted = st.verify_round()
        n, b = replay_round(f"{cfg.name} {kind} K={K} round {r}", st, None if draft is None else draft.stage, s, ctr0,
                            drafts, emitted, errors, overlap)
        band += b
        kept += n
        n_drafts += len(drafts)
    print(f"{cfg.name} {kind} K={K}: {kept} of {n_drafts} drafts kept, {band} in-band cases")
    assert not errors, "\n".join(errors[:10])
    assert band <= 2
    if kind == "same":
        # the assistant is the model: its rows equal the target's up to the paths' last bf16 bits (which can move a
        # near tie across the top-k boundary of a row), so a draft is kept with probability >= 0.95 on average (here
        # from the rows themselves); the count itself is random, with one rejection of slack for the 8 drafts at K = 1
        assert np.mean(overlap) >= 0.95, overlap
        assert kept >= 0.95 * n_drafts - 1
    if kind == "lookup":
        assert n_drafts > 0


@pytest.mark.parametrize("kind", ["same", "other_seed", "two_layers", "lookup"])
def test_graph_eager_and_seeds(kind):
    cfg = C.TINY_QWEN2_D128
    dm, draft = _target(cfg), _assistant(cfg, kind)
    ids = _prompt(cfg, kind)
    kw = dict(max_new_tokens=40, do_sample=True, top_k=8, temperature=0.9, top_p=0.95)
    kw.update(assistant_model=draft, num_assistant_tokens=3) if draft is not None else kw.update(prompt_lookup_num_tokens=3)
    greedy = dm.generate(ids, max_new_tokens=40).cpu()
    a = dm.generate(ids, seed=7, **kw).cpu()
    assert torch.equal(dm.generate(ids, seed=7, **kw).cpu(), a)                  # the same seed, the same tokens
    assert torch.equal(dm.generate(ids, seed=7, use_graph=False, **kw).cpu(), a)  # graph == eager, bit for bit
    assert not torch.equal(dm.generate(ids, seed=8, **kw).cpu(), a)
    assert torch.equal(dm.generate(ids, max_new_tokens=40).cpu(), greedy)        # greedy is left as it was
    assert a.shape == (1, ids.shape[1] + 40) and torch.equal(a[:, :ids.shape[1]], ids)


# ------------------------------------------------------------------------------------------ 4. generate's distribution
def _warped(logits_row, s):
    rm = sample_row_model(logits_row.bfloat16(), s["temperature"], s["top_k"], s["top_p"])
    return rm.w / rm.w.sum()


TOPK_GAP = 0.05       # the teacher-forced k-th and (k+1)-th logits lie further apart than the paths' rounding


def _law(dm, ids, s):
    """p(t1) p(t2|t1) p(t3|t1,t2) from the CUDA stage's own teacher-forced logits, warped by the sampler's rules; None
    when a top-k boundary is too close to call (the forward and the decode / verify paths round the logits differently,
    and a near tie there moves a token in or out of the kept set)"""
    def warped(seq):
        row = dm(seq).logits[0, -1].float().cpu()
        top = row.topk(s["top_k"] + 1).values
        return _warped(row, s) if float(top[-2] - top[-1]) > TOPK_GAP else None

    law = {}
    p1 = warped(ids)
    if p1 is None:
        return None
    for t1 in np.nonzero(p1)[0]:
        seq1 = torch.cat([ids, torch.tensor([[t1]])], dim=1)
        p2 = warped(seq1)
        if p2 is None:
            return None
        for t2 in np.nonzero(p2)[0]:
            p3 = warped(torch.cat([seq1, torch.tensor([[t2]])], dim=1))
            if p3 is None:
                return None
            for t3 in np.nonzero(p3)[0]:
                law[(int(t1), int(t2), int(t3))] = p1[t1] * p2[t2] * p3[t3]
    return law


@pytest.mark.parametrize("kind", ["same", "other_seed", "lookup"])
def test_generate_distribution(kind):
    cfg = C.TINY_QWEN2
    dm, draft = _target(cfg), _assistant(cfg, kind)
    s = _sampling(0, top_k=2)                         # top-2: few enough conditionals that a prompt with every one clear exists
    for seed in range(200):                           # the first prompt whose every top-k boundary is clear
        ids = synthetic_tokens(cfg, 1, 12, seed=seed)
        if kind == "lookup":
            ids = ids[:, :5].repeat(1, 3)
        law = _law(dm, ids, s)
        if law is not None:
            break
    assert law is not None, "no prompt with clear top-k boundaries"
    S, N = ids.shape[1], 4000
    kw = dict(max_new_tokens=3, do_sample=True, top_k=s["top_k"], use_graph=False)
    kw.update(assistant_model=draft, num_assistant_tokens=2) if draft is not None else kw.update(prompt_lookup_num_tokens=2)
    counts = {}
    for seed in range(N):
        t = tuple(dm.generate(ids, seed=seed, **kw)[0, S:].tolist())
        counts[t] = counts.get(t, 0) + 1
    outside = sum(c for k, c in counts.items() if k not in law)
    assert outside == 0, (outside, N)
    keys = sorted(law)
    ok, stat = _chi2_ok(np.array([counts.get(k, 0) for k in keys], float), np.array([law[k] for k in keys]) * N)
    print(f"{kind}: {len(counts)} triples seen of {len(law)}, chi2 {stat}, {outside} outside the law")
    assert ok, stat


def test_boundaries_and_streamer():
    """max_new_tokens and EOS cut a sampled assisted run where it would stop anyway (the rounds are the same), and the
    streamer sees exactly the result; with prompt lookup the run ends at its first EOS."""
    cfg = C.TINY_QWEN2
    dm, draft = _target(cfg), _assistant(cfg, "two_layers")
    ids = _prompt(cfg, "two_layers")
    S = ids.shape[1]
    kw = dict(do_sample=True, seed=5, top_k=6, assistant_model=draft, num_assistant_tokens=4)
    full = dm.generate(ids, max_new_tokens=30, **kw).cpu()
    for m in (1, 2, 4, 5, 6, 29):
        got = dm.generate(ids, max_new_tokens=m, **kw).cpu()
        assert torch.equal(got, full[:, :S + m]), m
    j = next(s for s in range(3, 30) if int(full[0, S + s]) not in full[0, S:S + s].tolist())
    eos = int(full[0, S + j])
    got = dm.generate(ids, max_new_tokens=30, eos_token_id=eos, **kw).cpu()
    assert torch.equal(got, apply_eos(full, S, eos)) and got.shape[1] == S + j + 1

    class _Streamer:
        def __init__(self):
            self.puts, self.ended = [], False

        def put(self, t):
            self.puts.append(t.clone())

        def end(self):
            self.ended = True

    for extra in (dict(assistant_model=draft, num_assistant_tokens=3), dict(prompt_lookup_num_tokens=3)):
        st = _Streamer()
        args = dict(do_sample=True, seed=9, top_k=6, max_new_tokens=25, **extra)
        got = dm.generate(ids, streamer=st, **args).cpu()
        assert st.ended and torch.cat(st.puts).tolist() == got[0, S:].tolist()
        # (with prompt lookup the EOS id also cuts the device's drafts, so the draws after it may differ)
        eos = int(got[0, S + 5])
        cut = dm.generate(ids, eos_token_id=eos, **args).cpu()[0, S:].tolist()
        assert (cut[-1] == eos and eos not in cut[:-1]) if eos in cut else len(cut) == 25


# ------------------------------------------------------------------------------------------ 5. vocabularies, full size
@pytest.mark.parametrize("vq", ["half", "double"])
def test_mismatched_vocabularies(vq):
    cfg = C.TINY_QWEN2
    dm = _target(cfg)
    draft = _make(cfg.scaled(vocab=cfg.vocab // 2 if vq == "half" else cfg.vocab * 2, n_layers=2))
    ids = synthetic_tokens(cfg, 1, 16)
    ids[0, ::2] = cfg.vocab // 2 + torch.arange(8)                # ids a half-size assistant cannot embed
    s = _sampling(31, top_k=0)
    _begin(dm, draft, ids, 4, s, 40)
    errors, band = [], 0
    for r in range(6):
        ctr0 = dm.stage.pl["ctr"].cpu().numpy().astype(np.int64)
        drafts, emitted = dm.stage.verify_round()
        band += replay_round(f"{vq} round {r}", dm.stage, draft.stage, s, ctr0, drafts, emitted, errors)[1]
    assert not errors, "\n".join(errors[:10])
    kw = dict(max_new_tokens=32, do_sample=True, seed=3, top_k=0, assistant_model=draft, num_assistant_tokens=4)
    got = dm.generate(ids, **kw).cpu()
    assert torch.equal(dm.generate(ids, use_graph=False, **kw).cpu(), got)
    assert int(got.max()) < cfg.vocab


def test_full_size_qwen25_7b_with_05b_assistant():
    """Qwen2.5-7B (V = 152,064) with a Qwen2.5-0.5B assistant (V = 151,936), device-initialised weights, sampled."""
    dm = _make(C.QWEN25_7B, init="device")
    draft = _make(C.QWEN25_05B, init="device")
    ids = synthetic_tokens(C.QWEN25_7B, 1, 32)
    for K in (2, 5):
        kw = dict(max_new_tokens=40, do_sample=True, seed=11, assistant_model=draft, num_assistant_tokens=K)
        got = dm.generate(ids, **kw).cpu()
        steps = dm.timers["assisted_steps"]
        assert torch.equal(dm.generate(ids, **kw).cpu(), got)
        assert torch.equal(dm.generate(ids, use_graph=False, **kw).cpu(), got)
        assert int(got.max()) < C.QWEN25_7B.vocab and got.shape == (1, 72)
        print(f"Qwen2.5-7B + 0.5B sampled K={K}: 40 tokens in {steps} rounds")
    del dm, draft
    torch.cuda.empty_cache()
