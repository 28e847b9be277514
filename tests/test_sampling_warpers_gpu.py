"""min_p / typical_p / epsilon_cutoff / eta_cutoff on the device: tl_sample and tl_sample_proc draw by draw against the
float64 row model (tests/warpers_model.py) and its Philox stream, the logged scores, neutral arguments, HF's law,
speculative acceptance, and generate end to end in every sampled mode."""
import functools

import numpy as np
import pytest
import torch

from tensorlink_b200.ml import configs as C
from tensorlink_b200.ml.weights import synthetic_tokens
from tests.rowwise_cases import check_draws, philox_u, sample_row_model
from tests.test_spec_sampling_gpu import DRAW_ROW, _chi2_ok, spec_replay
from tests.warpers_model import Warp, hf_warped, processed_values, warped_model

pytestmark = pytest.mark.gpu

SEED = 0x5EED_0001_2345
N = 2000


@pytest.fixture(scope="module")
def nat():
    from tensorlink_b200 import native
    native.require_device()
    return native


def _row(V, seed, scale=2.5):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(V, generator=g) * scale).to(torch.bfloat16)


def _argmax_dropper(V=48):
    x = torch.full((V,), 0.0)
    x[0] = 6.0
    x[1:21] = 3.0
    return x.to(torch.bfloat16)


WARPS = {"min_p": Warp(min_p=0.08), "min_p1": Warp(min_p=1.0), "typical": Warp(typical_p=0.6),
         "epsilon": Warp(epsilon=3e-3), "eta": Warp(eta=2e-3), "chain": Warp(min_p=0.02, typical_p=0.9, epsilon=1e-4, eta=3e-4)}
# name, V, temperature, top_k, top_p, warp, row maker
CASES = [(f"{w}.V{V}.T{T}", V, T, k, p, WARPS[w], None)
         for w in WARPS for (V, T, k, p) in ((1000, 0.7, 0, 1.0), (151_936, 1.0, 50, 0.95), (48, 20.0, 0, 1.0))]
CASES.append(("typical_drops_argmax", 48, 1.0, 0, 1.0, Warp(typical_p=0.3), _argmax_dropper))


def _inputs(case, i):
    name, V, T, k, p, w, maker = case
    return maker() if maker else _row(V, 97 * i + V)


def _history(nat, V, prompt):
    L = 64
    log = torch.zeros(1, L, dtype=torch.int32, device="cuda")
    ln = torch.zeros(1, dtype=torch.int32, device="cuda")
    bt = torch.zeros(1, (V + 31) // 32, dtype=torch.int32, device="cuda")
    nat.history_fill(prompt.cuda().view(1, -1).contiguous(), log, ln, bt, V)
    return log, ln, bt


def _draws(nat, row, case, proc, log_cols=0, explicit_neutral=False):
    """N draws of one row (fresh counter 0..N-1), with the score log of the first log_cols draws"""
    name, V, T, k, p, w, _ = case
    lg = row.view(1, -1).cuda()
    ids = torch.empty(1, dtype=torch.int64, device="cuda")
    ctr = torch.zeros(1, dtype=torch.int32, device="cuda")
    kw = w.kwargs() if not explicit_neutral else Warp().kwargs()
    if explicit_neutral is None:
        kw = {}
    out, logs = [], None
    if log_cols:
        raw = torch.full((log_cols, 1, V), 7.0, device="cuda")
        sc = torch.full((log_cols, 1, V), 7.0, device="cuda")
        col = torch.zeros(2, dtype=torch.int32, device="cuda")
        logs = (raw, sc, col, 0)
    prompt = torch.arange(0, V, max(1, V // 20))[:20]
    if proc:
        log, ln, bt = _history(nat, V, prompt)
        ln0, bt0 = ln.clone(), bt.clone()
        params = nat.lp_params(1.3, 0, 0, prompt.numel(), []).cuda()
        ws = torch.empty(nat.logits_proc_ws(1, V), dtype=torch.uint8, device="cuda")
    else:
        ws = torch.empty(nat.sample_ws(1), dtype=torch.uint8, device="cuda")
    for t in range(N):
        lgd = logs if (logs is not None and t < log_cols) else None
        if proc:
            nat.sample_proc(lg, ids, log, ln, bt, params, ctr, ws, T, k, p, SEED, 0, score_log=lgd, **kw)
            ln.copy_(ln0)
            bt.copy_(bt0)
        else:
            nat.sample(lg, ids, ctr, ws, T, k, p, SEED, log=lgd, **kw)
        out.append(ids.clone())
    assert int(ctr.item()) == N
    return torch.cat(out).cpu().numpy(), logs, prompt


def _model(row, case, proc, prompt):
    name, V, T, k, p, w, _ = case
    present = None
    if proc:
        present = np.zeros(V, bool)
        present[prompt.numpy()] = True
    return warped_model(row, T, k, p, w, proc=proc, present=present, penalty=1.3), present


@pytest.mark.parametrize("proc", [False, True], ids=["bf16", "proc"])
@pytest.mark.parametrize("case", CASES, ids=lambda c: c[0])
def test_draw_by_draw_and_logged_scores(nat, case, proc):
    row = _inputs(case, CASES.index(case))
    got, logs, prompt = _draws(nat, row, case, proc, log_cols=2)
    rm, present = _model(row, case, proc, prompt)
    assert rm.pinned, "a warper boundary lies inside its error band (case not pinned)"
    errors = []
    band = check_draws(case[0], got, rm, philox_u(SEED, 0, np.arange(N)), errors)
    assert not errors, "\n".join(errors[:5])
    assert band <= N // 50
    # the log: x / T (IEEE division) on the model's kept set, -inf elsewhere; the ids equal the unlogged run's
    raw, sc, col, _ = logs
    x = processed_values(row, present, None, 1.3) if proc else row.float().numpy()
    want = np.where(rm.kept, (torch.from_numpy(x) / torch.tensor(case[2], dtype=torch.float32)).numpy(), -np.inf)
    for c in range(2):
        assert np.array_equal(sc[c, 0].cpu().numpy(), want.astype(np.float32))
        assert torch.equal(raw[c, 0].cpu(), row.float())
    plain, _, _ = _draws(nat, row, case, proc)
    assert np.array_equal(plain, got)


@pytest.mark.parametrize("proc", [False, True], ids=["bf16", "proc"])
def test_neutral_arguments_keep_the_sampler_as_it_was(nat, proc):
    """(0, 1, 0, 0) passed to the C entry points, explicitly and by default: the draws follow the top-k / top-p rule of
    rowwise_cases.sample_row_model (the sampler without the warpers) draw by draw, and the score log is x / T on that
    rule's kept set; the ids, counters and logs of both calls are identical"""
    case = ("neutral", 1000, 0.7, 40, 0.9, Warp(), None)
    row = _row(1000, 5)
    a, la, prompt = _draws(nat, row, case, proc, log_cols=3, explicit_neutral=None)
    b, lb, _ = _draws(nat, row, case, proc, log_cols=3, explicit_neutral=True)
    assert np.array_equal(a, b)
    for x, y in zip(la[:3], lb[:3]):
        assert torch.equal(x, y)
    present = None
    if proc:
        present = np.zeros(1000, bool)
        present[prompt.numpy()] = True
    rm = sample_row_model(row, 0.7, 40, 0.9, proc=proc, present=present, penalty=1.3)
    assert rm.pinned
    errors = []
    assert check_draws("neutral", a, rm, philox_u(SEED, 0, np.arange(N)), errors) <= N // 50
    assert not errors, "\n".join(errors[:5])
    x = processed_values(row, present, None, 1.3) if proc else row.float().numpy()
    want = np.where(rm.kept, (torch.from_numpy(x) / torch.tensor(0.7, dtype=torch.float32)).numpy(), -np.inf)
    assert np.array_equal(la[1][0, 0].cpu().numpy(), want.astype(np.float32))


def test_out_of_range_warpers_are_rejected(nat):
    """values outside 0 <= min_p <= 1, 0 < typical_p <= 1, 0 <= epsilon < 1, 0 <= eta < 1 fail with TL_ERR_INVALID
    (no launch); the range ends that are inside run"""
    lg = _row(64, 1).view(1, -1).cuda()
    ids = torch.empty(1, dtype=torch.int64, device="cuda")
    ctr = torch.zeros(1, dtype=torch.int32, device="cuda")
    ws = torch.empty(nat.sample_ws(1), dtype=torch.uint8, device="cuda")
    for bad in (dict(min_p=-0.01), dict(min_p=1.01), dict(typical_p=0.0), dict(typical_p=1.01), dict(epsilon=1.0),
                dict(epsilon=-0.1), dict(eta=1.0), dict(eta=-1e-3), dict(min_p=float("nan"))):
        with pytest.raises(nat.NativeError):
            nat.sample(lg, ids, ctr, ws, 1.0, 0, 1.0, SEED, **bad)
    assert int(ctr.item()) == 0
    nat.sample(lg, ids, ctr, ws, 1.0, 0, 1.0, SEED, min_p=1.0, typical_p=1.0, epsilon=0.0, eta=0.0)
    assert int(ctr.item()) == 1 and int(ids.item()) == int(torch.argmax(lg[0].float()))


# ------------------------------------------------------------------------------------------ banned ids (-inf values)
def _ban_setup(row, V, ban):
    """a history of the row's 10 largest logits and 10 others, and the processor parameters: no_repeat_ngram_size=1
    bans every id of it; min_new_tokens with EOS ids bans those (the top logit among them).  Returns the device
    parameters and HF's view: the processed fp32 values with -inf on the banned ids"""
    from transformers.generation import logits_process as L
    top = torch.topk(row.float(), 10).indices
    prompt = torch.cat([top, torch.arange(1, 11) * (V // 11)])
    eos = [int(top[0]), int(top[3]), 2]
    ngram, min_new = (1, 0) if ban == "ngram" else (0, 100)
    hist = prompt.view(1, -1)
    x = L.RepetitionPenaltyLogitsProcessor(1.3)(hist, row.float()[None].clone())
    if ngram:
        x = L.NoRepeatNGramLogitsProcessor(ngram)(hist, x)
    if min_new:
        x = L.MinNewTokensLengthLogitsProcessor(prompt.numel(), min_new, eos)(hist, x)
    return prompt, nat_params(ngram, min_new, prompt.numel(), eos if min_new else []), x[0]


def nat_params(ngram, min_new, prompt_len, eos):
    from tensorlink_b200 import native
    return native.lp_params(1.3, ngram, min_new, prompt_len, eos).cuda()


BAN_WARPS = {"typical": Warp(typical_p=0.6), "eta": Warp(eta=2e-3), "chain": Warp(min_p=0.02, typical_p=0.9, eta=3e-4)}


@pytest.mark.parametrize("V", [1000, 151_936])
@pytest.mark.parametrize("ban", ["ngram", "min_new"])
@pytest.mark.parametrize("wname", list(BAN_WARPS))
def test_banned_ids_with_top_k_off(nat, wname, ban, V):
    """top_k = 0, top_p = 1: the banned ids (-inf) lie inside the kept interval's keys, and weigh nothing in the
    entropy of typical and eta; draw by draw against the model, and the kept set equals HF's chain"""
    T, w = 0.8, BAN_WARPS[wname]
    row = _row(V, 3 * V + len(wname) + len(ban))
    prompt, params, xh = _ban_setup(row, V, ban)
    log, ln, bt = _history(nat, V, prompt)
    ln0, bt0 = ln.clone(), bt.clone()
    lg = row.view(1, -1).cuda()
    ids = torch.empty(1, dtype=torch.int64, device="cuda")
    ctr = torch.zeros(1, dtype=torch.int32, device="cuda")
    ws = torch.empty(nat.logits_proc_ws(1, V), dtype=torch.uint8, device="cuda")
    got = []
    for _ in range(N):
        nat.sample_proc(lg, ids, log, ln, bt, params, ctr, ws, T, 0, 1.0, SEED, nat.LP_BAN, **w.kwargs())
        ln.copy_(ln0)
        bt.copy_(bt0)
        got.append(ids.clone())
    got = torch.cat(got).cpu().numpy()
    present = np.zeros(V, bool)
    present[prompt.numpy()] = True
    banned = ~torch.isfinite(xh).numpy()
    assert banned.sum() >= 3
    rm = warped_model(row, T, 0, 1.0, w, proc=True, present=present, banned=banned, penalty=1.3)
    assert rm.pinned, "a warper boundary lies inside its error band (case not pinned)"
    hf = torch.isfinite(hf_warped(xh[None], T, 0, 1.0, w))[0].numpy()
    assert np.array_equal(rm.kept, hf), "the model's kept set differs from HF's"
    assert not rm.kept[banned].any()
    errors = []
    band = check_draws(f"{wname}.{ban}.V{V}", got, rm, philox_u(SEED, 0, np.arange(N)), errors)
    assert not errors, "\n".join(errors[:5])
    # the band grows with the kept set's summed weight errors: thousands of kept ids at V = 151,936 with top-k off
    assert band <= (N // 50 if rm.kept.sum() < 1000 else N // 10), band


def test_hf_law(nat):
    """the support lies within HF's warped set and 20,000 draws follow HF's warped softmax"""
    case = ("law", 1000, 0.8, 0, 0.97, Warp(min_p=0.01, typical_p=0.95, epsilon=2e-4, eta=1e-3), None)
    row = _row(1000, 11, scale=1.5)
    hf = hf_warped(row.float()[None], 0.8, 0, 0.97, case[5])[0]
    prob = torch.softmax(hf.double(), -1).numpy()
    lg = row.view(1, -1).cuda()
    ids = torch.empty(1, dtype=torch.int64, device="cuda")
    ctr = torch.zeros(1, dtype=torch.int32, device="cuda")
    ws = torch.empty(nat.sample_ws(1), dtype=torch.uint8, device="cuda")
    got = []
    for _ in range(20_000):
        nat.sample(lg, ids, ctr, ws, 0.8, 0, 0.97, SEED, **case[5].kwargs())
        got.append(ids.clone())
    got = torch.cat(got).cpu().numpy()
    assert np.isfinite(hf.numpy()[got]).all(), "a draw outside HF's warped set"
    ok, stat = _chi2_ok(np.bincount(got, minlength=1000).astype(np.float64), prob * len(got))
    assert ok, stat


def test_spec_accept_with_warpers(nat):
    """tl_spec_accept with the warpers: every step against the replay of its rule, and the emitted tokens follow the
    target's warped row (chi-square)"""
    K, V, T = 3, 1000, 0.9
    w = Warp(min_p=0.02, typical_p=0.9, eta=1e-3)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(K + 1, V, generator=g) * 2.0
    y = x[:K] + torch.randn(K, V, generator=g) * 0.8
    P, Q = x.to(torch.bfloat16), y.to(torch.bfloat16)
    pm = [warped_model(P[i], T, 0, 1.0, w) for i in range(K + 1)]
    qm = [warped_model(Q[i], T, 0, 1.0, w) for i in range(K)]
    assert all(m.pinned for m in pm + qm)
    ws = torch.empty(nat.spec_accept_ws(K), dtype=torch.uint8, device="cuda")
    Pd, Qd = P.cuda(), Q.cuda()
    seed, rng, errors, band, first = 0xABCDEF, np.random.default_rng(1), [], 0, []
    for t in range(400):
        drafts = []
        for i in range(K):
            wq = qm[i].w / qm[i].w.sum()
            drafts.append(int(rng.choice(V, p=wq)))
        in_ids = torch.tensor([5] + drafts, dtype=torch.int64, device="cuda")
        n_cand = torch.tensor([K], dtype=torch.int32, device="cuda")
        ctr = torch.tensor([t], dtype=torch.int32, device="cuda")
        ids = torch.full((K + 1,), -7, dtype=torch.int64, device="cuda")
        nat.spec_accept(Pd, Qd, in_ids, n_cand, ctr, ids, ws, T, 0, 1.0, seed, **w.kwargs())
        got = ids.cpu().tolist()
        u_acc = [float(philox_u(seed, i, [t])[0]) for i in range(K)]
        n, b = spec_replay(f"step {t}", pm, qm, drafts, u_acc, float(philox_u(seed, DRAW_ROW, [t])[0]), got, errors)
        band += b
        first.append(got[0])
    assert not errors, "\n".join(errors[:5])
    assert band <= 20
    # the first emitted token of every step follows p_0 (speculative sampling's guarantee)
    p0 = pm[0].w / pm[0].w.sum()
    assert all(pm[0].kept[t] for t in first)
    ok, stat = _chi2_ok(np.bincount(first, minlength=V).astype(np.float64), p0 * len(first))
    assert ok, stat


# ------------------------------------------------------------------------------------------ generate
@functools.lru_cache(maxsize=None)
def _dm(cfg, max_batch=2):
    from tensorlink_b200.ml import DistributedModel
    return DistributedModel(cfg, training=False, max_batch=max_batch, max_seq=128, seed=1234)


GEN_WARPS = {"min_p": dict(min_p=0.1), "typical": dict(typical_p=0.7), "epsilon": dict(epsilon_cutoff=2e-3),
             "eta": dict(eta_cutoff=3e-3), "chain": dict(min_p=0.02, typical_p=0.9, epsilon_cutoff=1e-4, eta_cutoff=5e-4)}


def _hf_pattern(dm, ids, out, kw, T, top_k, procs=None):
    """every column's -inf pattern against HF's warper chain on that column's logits (after HF's processors on the
    history: ``procs`` = generate's repetition_penalty / no_repeat_ngram_size / min_new_tokens / eos_token_id);
    returns the number of pinned rows that differ"""
    from transformers.generation import logits_process as L
    procs = procs or {}
    w = Warp(kw.get("min_p", 0.0), kw.get("typical_p", 1.0), kw.get("epsilon_cutoff", 0.0), kw.get("eta_cutoff", 0.0))
    penalty = procs.get("repetition_penalty")
    S = ids.shape[1]
    bad = 0
    for c, (sc, lg) in enumerate(zip(out.scores, out.logits)):
        hist = out.sequences[:, :S + c].cpu()
        x = lg.cpu().float()
        if penalty:
            x = L.RepetitionPenaltyLogitsProcessor(penalty)(hist, x)
        if procs.get("no_repeat_ngram_size"):
            x = L.NoRepeatNGramLogitsProcessor(procs["no_repeat_ngram_size"])(hist, x)
        if procs.get("min_new_tokens"):
            x = L.MinNewTokensLengthLogitsProcessor(S, procs["min_new_tokens"], [procs["eos_token_id"]])(hist, x)
        hf = torch.isfinite(hf_warped(x, T, top_k, 1.0, w))
        dev = torch.isfinite(sc.cpu())
        for r in range(x.shape[0]):
            if torch.equal(hf[r], dev[r]):
                continue
            proc = bool(procs)
            rm = warped_model(lg[r].cpu().to(torch.bfloat16), T, top_k, 1.0, w, proc=proc,
                              present=np.isin(np.arange(x.shape[1]), hist[r].numpy()) if penalty else None,
                              banned=(~torch.isfinite(x[r])).numpy() if proc else None, penalty=penalty or 1.0)
            bad += rm.pinned
    return bad


@pytest.mark.parametrize("cfg", [C.TINY_QWEN2, C.TINY_QWEN3], ids=lambda c: c.name)
@pytest.mark.parametrize("wname", list(GEN_WARPS))
def test_generate_scores_follow_hf(cfg, wname):
    dm = _dm(cfg)
    ids = synthetic_tokens(cfg, 2, 8)
    kw = GEN_WARPS[wname]
    for pen in (None, 1.3):
        extra = {} if pen is None else dict(repetition_penalty=pen)
        out = dm.generate(ids.cuda(), max_new_tokens=6, do_sample=True, temperature=0.9, top_k=0, seed=7,
                          return_dict_in_generate=True, output_scores=True, output_logits=True, **kw, **extra)
        assert _hf_pattern(dm, ids, out, kw, 0.9, 0, extra) == 0
        again = dm.generate(ids.cuda(), max_new_tokens=6, do_sample=True, temperature=0.9, top_k=0, seed=7, **kw, **extra)
        assert torch.equal(again.cpu(), out.sequences.cpu()), "a seed reproduces its tokens"
        eager = dm.generate(ids.cuda(), max_new_tokens=6, do_sample=True, temperature=0.9, top_k=0, seed=7,
                            use_graph=False, **kw, **extra)
        assert torch.equal(eager.cpu(), out.sequences.cpu()), "graph and eager runs agree"


@pytest.mark.parametrize("wname", ["typical", "eta", "chain"])
def test_generate_scores_with_bans_follow_hf(wname):
    """no_repeat_ngram_size and min_new_tokens put -inf values inside the kept interval (top_k = 0): every column's
    scores still follow HF's processors and warper chain"""
    cfg = C.TINY_QWEN2
    dm = _dm(cfg)
    ids = synthetic_tokens(cfg, 2, 8)
    ids[:, 4:] = ids[:, :4]                          # repeated bigrams: the n-gram rule bans ids from the first step
    eos = int(ids[0, 1])
    procs = dict(no_repeat_ngram_size=2, min_new_tokens=6, eos_token_id=eos, repetition_penalty=1.2)
    kw = GEN_WARPS[wname]
    out = dm.generate(ids.cuda(), max_new_tokens=6, do_sample=True, temperature=0.9, top_k=0, seed=9,
                      return_dict_in_generate=True, output_scores=True, output_logits=True, **kw, **procs)
    assert any(bool(torch.isinf(sc).any()) for sc in out.scores)
    assert _hf_pattern(dm, ids, out, kw, 0.9, 0, procs) == 0


def test_generate_left_padded_batch():
    cfg = C.TINY_QWEN2
    dm = _dm(cfg)
    ids = synthetic_tokens(cfg, 2, 8)
    mask = torch.ones_like(ids)
    mask[1, :3] = 0
    ids[1, :3] = 0
    got = dm.generate(ids.cuda(), attention_mask=mask.cuda(), max_new_tokens=5, do_sample=True, seed=3,
                      **GEN_WARPS["chain"])
    assert got.shape == (2, 13)
    again = dm.generate(ids.cuda(), attention_mask=mask.cuda(), max_new_tokens=5, do_sample=True, seed=3,
                        **GEN_WARPS["chain"])
    assert torch.equal(got.cpu(), again.cpu())


def test_sharp_warpers_reproduce_greedy_in_every_sampled_mode():
    """min_p = 1 (and epsilon near 1) keep only the top token on rows without a top-2 tie: sampled decode, sampled
    prompt lookup and sampled assisted decoding each give greedy decoding's tokens"""
    from tensorlink_b200.ml import DistributedModel
    cfg = C.TINY_QWEN2
    dm = DistributedModel(cfg, training=False, max_batch=1, max_seq=128, seed=1234)
    asst = DistributedModel(cfg.scaled(n_layers=2), training=False, max_batch=1, max_seq=128, seed=1234)
    ids = synthetic_tokens(cfg, 1, 12)[:, :5].repeat(1, 3).cuda()       # self-repeating: the lookup finds drafts
    greedy = dm.generate(ids, max_new_tokens=12, return_dict_in_generate=True, output_logits=True)
    for lg in greedy.logits:                                              # no top-2 tie on the greedy path
        top2 = torch.topk(lg[0].float(), 2).values
        assert top2[0] > top2[1]
    want = greedy.sequences.cpu()
    for sharp in (dict(min_p=1.0), dict(epsilon_cutoff=0.999999)):
        for mode in ({}, dict(prompt_lookup_num_tokens=3), dict(assistant_model=asst, num_assistant_tokens=3)):
            got = dm.generate(ids, max_new_tokens=12, do_sample=True, temperature=1.0, top_k=0, seed=11, **sharp, **mode)
            assert torch.equal(got.cpu(), want), (sharp, list(mode))
