"""Logits processors on the device (csrc/logits_process.cu, the processed argmax in lmhead.cu, the processed sampler in
sample.cu) against HF's own RepetitionPenaltyLogitsProcessor -> NoRepeatNGramLogitsProcessor ->
MinNewTokensLengthLogitsProcessor on the fp32 copy of the same bf16 logits, and ``DistributedModel.generate`` with
``repetition_penalty`` / ``no_repeat_ngram_size`` / ``min_new_tokens`` against HF ``generate`` on the same weights."""
import pytest
import torch

from tensorlink_b200.ml import configs as C
from tensorlink_b200.ml import module as M
from tensorlink_b200.ml.weights import init_state_dict, synthetic_tokens

pytestmark = pytest.mark.gpu

MARGIN = 0.05


@pytest.fixture(scope="module")
def nat():
    from tensorlink_b200 import native
    native.require_device()
    return native


def hf_processed(logits_bf16, hist, penalty=1.0, ngram=0, min_new=0, prompt_len=0, eos=()):
    """HF's processed scores (fp32, CPU) for each row's history ``hist`` (list of int64 rows, any lengths)."""
    from transformers.generation.logits_process import (MinNewTokensLengthLogitsProcessor, NoRepeatNGramLogitsProcessor,
                                                        RepetitionPenaltyLogitsProcessor)
    out = []
    for r, h in enumerate(hist):
        s = logits_bf16[r:r + 1].float().clone()
        ids = h.view(1, -1)
        if penalty != 1.0:
            s = RepetitionPenaltyLogitsProcessor(penalty)(ids, s)
        if ngram:
            s = NoRepeatNGramLogitsProcessor(ngram)(ids, s)
        if min_new and eos:
            s = MinNewTokensLengthLogitsProcessor(prompt_len, min_new, list(eos))(ids, s)
        out.append(s)
    return torch.cat(out)


class Hist:
    """A device token history for M rows (the layout CudaStage keeps per slot)."""

    def __init__(self, nat, M, V, L):
        self.nat, self.V = nat, V
        self.log = torch.zeros(M, L, dtype=torch.int32, device="cuda")
        self.len = torch.zeros(M, dtype=torch.int32, device="cuda")
        self.bits = torch.zeros(M, (V + 31) // 32, dtype=torch.int32, device="cuda")
        self.ws = torch.empty(nat.logits_proc_ws(M, V), dtype=torch.uint8, device="cuda")

    def fill(self, prompt):
        self.nat.history_fill(prompt.cuda().contiguous(), self.log, self.len, self.bits, self.V)

    def params(self, penalty=1.0, ngram=0, min_new=0, prompt_len=0, eos=()):
        flags = self.nat.LP_BAN if ngram or (min_new and eos) else 0
        return self.nat.lp_params(penalty, ngram, min_new, prompt_len, list(eos) if min_new else []).cuda(), flags

    def read(self, m):
        n = int(self.len[m])
        bits = self.bits[m].cpu().view(torch.uint8).numpy()
        import numpy as np
        present = np.nonzero(np.unpackbits(bits, bitorder="little")[:self.V])[0].tolist()
        return self.log[m, :n].cpu().long(), present


def _history(g, M, V, lengths, pad):
    """int64 [M, S] prompts whose rows repeat tokens from a small pool, with a run of pad ids in front."""
    S = max(lengths)
    rows = torch.full((M, S), pad, dtype=torch.int64)
    for m in range(M):
        L = lengths[m % len(lengths)]
        pool = torch.randint(0, V, (max(2, L // 3),), generator=g)
        rows[m, S - L:] = pool[torch.randint(0, pool.numel(), (L,), generator=g)]
    return rows


def _tie(penalty):
    """(x, t): bf16 values with fp32(x / penalty) == t, t above every random logit of the tests."""
    for i in range(2000):
        x = torch.tensor(40.0 + 0.125 * i).bfloat16().float()
        q = x / penalty
        if float(q) > 30 and float(q.bfloat16().float()) == float(q):
            return float(x), float(q)
    raise AssertionError(f"no tie for penalty {penalty}")


ARGMAX_CASES = [  # V, penalty, ngram, min_new, history lengths
    (1000, 1.3, 0, 0, (1, 7, 40)),
    (1000, 0.7, 2, 0, (300, 5, 1)),
    (1000, 2.0, 1, 3, (64, 2, 17)),
    (1000, 1.3, 4, 0, (4096, 1024, 9)),
    (151936, 1.3, 3, 2, (4096, 77, 1)),
    (151936, 0.7, 0, 0, (2000, 3, 600)),
    (151936, 2.0, 2, 0, (12, 3000, 256)),
]


@pytest.mark.parametrize("V,penalty,ngram,min_new,lengths", ARGMAX_CASES)
def test_processed_argmax_equals_hf(nat, V, penalty, ngram, min_new, lengths):
    g = torch.Generator().manual_seed(V + len(lengths) + ngram)
    M, pad = 3, 5
    prompt = _history(g, M, V, lengths, pad)
    eos = (int(prompt[0, -1]), 11, V - 1)
    logits = (torch.randn(M, V, generator=g) * 3).bfloat16()
    # constructed ties at the top: a penalised value x / penalty equal to an unpenalised bf16 value t, the unpenalised
    # token at a lower index (row 0) or a higher one (row 1)
    x, t = _tie(penalty)
    for m in range(2):
        present = sorted(set(prompt[m].tolist()) - set(eos))
        absent = sorted(set(range(V)) - set(prompt[m].tolist()) - set(eos))
        a, b = present[len(present) // 2], (absent[0] if m == 0 else absent[-1])
        logits[m, a], logits[m, b] = x, t
    h = Hist(nat, M, V, prompt.shape[1] + 4)
    h.fill(prompt)
    params, flags = h.params(penalty, ngram, min_new, prompt.shape[1], eos)
    ids = torch.empty(M, dtype=torch.int64, device="cuda")
    hist = [prompt[m] for m in range(M)]
    for step in range(3):
        nat.argmax_proc(logits.cuda(), ids, h.log, h.len, h.bits, params, h.ws, flags)
        want = hf_processed(logits, hist, penalty, ngram, min_new, prompt.shape[1], eos).argmax(-1)
        assert torch.equal(ids.cpu(), want), (step, ids.cpu(), want)
        hist = [torch.cat([hist[m], want[m:m + 1]]) for m in range(M)]
    for m in range(M):
        log, present = h.read(m)
        assert torch.equal(log, hist[m])
        assert present == sorted(set(hist[m].tolist()))


def test_every_token_banned_gives_zero(nat):
    V = 1000
    prompt = torch.arange(V, dtype=torch.int64).flip(0).view(1, V)        # every id seen: n = 1 bans all of them
    logits = torch.randn(1, V, generator=torch.Generator().manual_seed(1)).bfloat16()
    h = Hist(nat, 1, V, V + 2)
    h.fill(prompt)
    params, flags = h.params(1.0, 1)
    ids = torch.full((1,), 7, dtype=torch.int64, device="cuda")
    nat.argmax_proc(logits.cuda(), ids, h.log, h.len, h.bits, params, h.ws, flags)
    assert int(ids) == 0 == int(hf_processed(logits, [prompt[0]], 1.0, 1).argmax(-1))
    ctr = torch.zeros(1, dtype=torch.int32, device="cuda")
    nat.sample_proc(logits.cuda(), ids, h.log, h.len, h.bits, params, ctr, h.ws, 1.0, 0, 0.9, 3, flags)
    assert int(ids) == 0 and int(ctr) == 1


def hf_warped(scores, temperature, top_k, top_p):
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    s = scores.clone()
    if temperature != 1.0:
        s = TemperatureLogitsWarper(temperature)(None, s)
    if top_k:
        s = TopKLogitsWarper(top_k)(None, s)
    if top_p < 1.0:
        s = TopPLogitsWarper(top_p)(None, s)
    return torch.softmax(s, -1)


def _draws(nat, logits_row, prompt_row, rows, iters, penalty, ngram, temperature, top_k, top_p, seed):
    """``rows`` identical rows (independent Philox streams) drawn ``iters`` times from a freshly filled history."""
    V = logits_row.shape[-1]
    lg = logits_row.view(1, V).expand(rows, V).contiguous().cuda()
    prompt = prompt_row.view(1, -1).expand(rows, -1).contiguous()
    h = Hist(nat, rows, V, prompt.shape[1] + 2)
    params, flags = h.params(penalty, ngram)
    ids = torch.empty(rows, dtype=torch.int64, device="cuda")
    ctr = torch.zeros(rows, dtype=torch.int32, device="cuda")
    out = []
    for _ in range(iters):
        h.fill(prompt)
        nat.sample_proc(lg, ids, h.log, h.len, h.bits, params, ctr, h.ws, temperature, top_k, top_p, seed, flags)
        out.append(ids.clone())
    assert ctr.cpu().tolist() == [iters] * rows
    log, _ = h.read(0)
    assert torch.equal(log, torch.cat([prompt_row, out[-1][:1].cpu()]))     # the draw joined the history
    return torch.stack(out, 1).cpu()


@pytest.mark.parametrize("penalty,ngram,temperature,top_k,top_p",
                         [(1.3, 0, 1.0, 0, 1.0), (0.7, 2, 0.8, 0, 1.0), (2.0, 1, 1.0, 6, 1.0), (1.3, 3, 1.2, 0, 0.7),
                          (1.3, 2, 0.9, 12, 0.9)])
def test_processed_sampling_frequencies(nat, penalty, ngram, temperature, top_k, top_p):
    g = torch.Generator().manual_seed(3)
    V = 48
    logits = (torch.randn(V, generator=g) * 2.0).bfloat16()
    prompt = torch.tensor([3, 9, 3, 17, 9, 3, 30, 9, 3], dtype=torch.int64)      # "9 3" repeats: n-gram bans
    probs = hf_warped(hf_processed(logits.view(1, V), [prompt], penalty, ngram), temperature, top_k, top_p)[0]
    ids = _draws(nat, logits, prompt, 50, 400, penalty, ngram, temperature, top_k, top_p, 1234).reshape(-1)
    n = ids.numel()
    counts = torch.bincount(ids, minlength=V).double()
    assert counts[probs == 0].sum() == 0, "a token outside HF's kept set was drawn"
    exp = probs.double() * n
    big = exp >= 5
    chi2 = float((((counts - exp) ** 2) / exp.clamp_min(1e-12))[big].sum())
    dof = int(big.sum()) - 1
    assert chi2 < dof + 6 * (2 * dof) ** 0.5 + 10, (chi2, dof)


def test_processed_sampling_full_vocabulary(nat):
    g = torch.Generator().manual_seed(6)
    V = 151936
    logits = (torch.randn(V, generator=g) * 1.5).bfloat16()
    prompt = torch.cat([logits.float().topk(40).indices, torch.tensor([1, 2, 1, 2])])   # penalise the top
    for kw in (dict(temperature=1.0, top_k=50, top_p=1.0), dict(temperature=0.9, top_k=0, top_p=0.8),
               dict(temperature=1.0, top_k=200, top_p=0.95)):
        scores = hf_processed(logits.view(1, V), [prompt], 1.3, 2)
        probs = hf_warped(scores, kw["temperature"], kw["top_k"], kw["top_p"])[0]
        ids = _draws(nat, logits, prompt, 8, 25, 1.3, 2, seed=9, **kw).reshape(-1)
        # HF's sort cuts inside a group of tied values at the top-p boundary, and which members survive depends on its
        # sort; the kernel keeps the whole group.  So the exact statement: every draw is at least HF's smallest survivor
        floor = scores[0][probs > 0].min()
        assert bool((scores[0][ids] >= floor).all()), kw


def test_processed_sampling_seed_and_counter(nat):
    g = torch.Generator().manual_seed(7)
    logits = (torch.randn(1000, generator=g) * 2.0).bfloat16()
    prompt = torch.randint(0, 1000, (30,), generator=g)
    a = _draws(nat, logits, prompt, 3, 32, 1.3, 2, 1.0, 0, 1.0, 42)
    b = _draws(nat, logits, prompt, 3, 32, 1.3, 2, 1.0, 0, 1.0, 42)
    c = _draws(nat, logits, prompt, 3, 32, 1.3, 2, 1.0, 0, 1.0, 43)
    assert torch.equal(a, b) and not torch.equal(a, c)
    assert len(set(a[0].tolist())) > 8 and not torch.equal(a[0], a[1])


# ------------------------------------------------------------------------------------------------- end to end
@pytest.fixture(scope="module")
def models():
    from tensorlink_b200.ml import DistributedModel
    from tests.hf_util import hf_model
    cache = {}

    def get(name, max_batch=12, n_pipelines=1):
        key = (name, max_batch, n_pipelines)
        cfg = getattr(C, name)
        if key not in cache:
            if (name, "hf") not in cache:
                hf = hf_model(cfg, init_state_dict(cfg))
                hf.generation_config.eos_token_id = None
                hf.generation_config.pad_token_id = 0
                cache[(name, "hf")] = hf
            cache[key] = DistributedModel(cfg, training=False, max_batch=max_batch, max_seq=256, n_pipelines=n_pipelines)
        return cfg, cache[key], cache[(name, "hf")]
    return get


def hf_generate(hf, ids, new, mask=None, **kw):
    out = hf.generate(ids, attention_mask=torch.ones_like(ids) if mask is None else mask, max_new_tokens=new,
                      do_sample=False, output_scores=True, return_dict_in_generate=True, **kw)
    sc = torch.stack(out.scores, 1).float()                       # [B, steps, V] processed scores
    top2 = sc.topk(2, -1).values
    return out.sequences, top2[..., 0] - top2[..., 1]


def check_ids(got, want, margins, S):
    """Exact up to each row's first step whose processed top-2 margin is below MARGIN (random weights give near-flat
    logits, so a row may have no such step); the number of steps checked."""
    n = 0
    for b in range(want.shape[0]):
        for s in range(min(margins.shape[1], got.shape[1] - S, want.shape[1] - S)):
            if margins[b, s] < MARGIN:
                break
            assert int(got[b, S + s]) == int(want[b, S + s]), (b, s, got[b, S:], want[b, S:])
            n += 1
    return n


def resolvable(make, seeds=range(40)):
    """The first ``make(seed)`` -> (want, margins, ...) whose first step HF resolves (top-2 margin >= MARGIN) in some row:
    random weights give near-flat logits, and a prompt whose every row is a close call would let a comparison check
    nothing."""
    for seed in seeds:
        got = make(seed)
        if bool((got[1][:, 0] >= MARGIN).any()):
            return got
    raise AssertionError("no prompt with a resolvable first step")


PROC_SETS = {"penalty": dict(repetition_penalty=1.3), "ngram": dict(no_repeat_ngram_size=2),
             "all": dict(repetition_penalty=1.2, no_repeat_ngram_size=3, min_new_tokens=4)}


@pytest.mark.parametrize("name", ["TINY_QWEN2", "TINY_QWEN3"])
@pytest.mark.parametrize("B", [1, 3, 12])
@pytest.mark.parametrize("procs", list(PROC_SETS))
def test_generate_matches_hf(models, name, B, procs):
    cfg, dm, hf = models(name)
    kw = PROC_SETS[procs]
    new = 20
    want, margins, ids = resolvable(lambda seed: (*hf_generate(hf, synthetic_tokens(cfg, B, 10, seed=seed), new, **kw),
                                                  synthetic_tokens(cfg, B, 10, seed=seed)), range(B, B + 40))
    got = dm.generate(ids, max_new_tokens=new, **kw).cpu()
    assert check_ids(got, want, margins, ids.shape[1]) >= 1
    if procs == "ngram":                                      # the HF guarantee itself: no bigram occurs twice
        for r in got.tolist():
            grams = list(zip(r, r[1:]))
            assert len(grams) == len(set(grams))
    if B == 3:
        eager = dm.generate(ids, max_new_tokens=new, use_graph=False, **kw).cpu()
        assert torch.equal(eager, got)


def test_micro_batches_equal_one(models):
    """n_pipelines=2 over 4 rows equals each half run as one micro-batch of 2 rows (the same decode path: GEMV)."""
    cfg, one, _ = models("TINY_QWEN2", 2, 1)
    _, two, _ = models("TINY_QWEN2", 4, 2)
    ids = synthetic_tokens(cfg, 4, 9, seed=3)
    kw = dict(max_new_tokens=16, repetition_penalty=1.3, no_repeat_ngram_size=2)
    halves = torch.cat([one.generate(ids[:2], **kw).cpu(), one.generate(ids[2:], **kw).cpu()])
    assert torch.equal(two.generate(ids, **kw).cpu(), halves)


def test_left_padded_pads_count_as_seen(models):
    cfg, dm, hf = models("TINY_QWEN2")
    lengths = (6, 11, 8)
    S = max(lengths) + 1                                             # one column that is pad in every row
    kw = dict(repetition_penalty=2.0)

    def make(seed):
        rows = [synthetic_tokens(cfg, 1, L, seed=seed + 10 * b) for b, L in enumerate(lengths)]
        pad = int(dm.generate(rows[0], max_new_tokens=1)[0, -1])   # row 0's unpenalised greedy next token
        ids = torch.full((3, S), pad, dtype=torch.int64)
        mask = torch.zeros(3, S, dtype=torch.int64)
        for b, (L, r) in enumerate(zip(lengths, rows)):
            ids[b, S - L:], mask[b, S - L:] = r[0], 1
        return (*hf_generate(hf, ids, 12, mask, **kw), ids, mask, pad)

    want, margins, ids, mask, pad = resolvable(make)
    got = dm.generate(ids, attention_mask=mask, max_new_tokens=12, pad_token_id=pad, **kw).cpu()
    assert check_ids(got, want, margins, S) >= 1
    # the pad id is penalised in every row, so row 0 no longer picks it first (its margin allowing)
    if margins[0, 0] >= MARGIN:
        assert int(got[0, S]) != pad


def test_min_new_tokens_holds_back_eos(models):
    cfg, dm, hf = models("TINY_QWEN3")

    def make(seed):
        ids = synthetic_tokens(cfg, 1, 10, seed=seed)
        plain = dm.generate(ids, max_new_tokens=16).cpu()
        eos = int(plain[0, 10 + 1])                                # emitted at the second step without the processor
        return (*hf_generate(hf, ids, 16, eos_token_id=eos, pad_token_id=eos, min_new_tokens=8), ids, plain, eos)

    want, margins, ids, plain, eos = resolvable(make, range(21, 61))
    first = [s for s in range(16) if int(plain[0, 10 + s]) == eos][0]
    cut = dm.generate(ids, max_new_tokens=16, eos_token_id=eos).cpu()
    assert cut.shape[1] == 10 + first + 1
    got = dm.generate(ids, max_new_tokens=16, eos_token_id=eos, min_new_tokens=8).cpu()
    assert check_ids(got, want, margins, 10) >= 1
    assert eos not in got[0, 10:18].tolist()


def test_two_penalties_and_neutral_values(models):
    cfg, dm, hf = models("TINY_QWEN2_D128")
    runs = {}

    def make(seed):                                               # a prompt HF resolves at the first step for both values
        ids = synthetic_tokens(cfg, 2, 12, seed=seed)
        runs.clear()
        runs.update({p: hf_generate(hf, ids, 16, repetition_penalty=p) for p in (1.5, 0.8)})
        ok = torch.minimum(runs[1.5][1][:, :1], runs[0.8][1][:, :1])
        return None, torch.cat([ok, ok], 1), ids

    _, _, ids = resolvable(make, range(8, 48))
    greedy = dm.generate(ids, max_new_tokens=16).cpu()
    sample_kw = dict(do_sample=True, temperature=0.9, top_k=20, top_p=0.95, seed=11, max_new_tokens=16)
    sampled = dm.generate(ids, **sample_kw).cpu()
    for p in (1.5, 0.8):                                          # the same captured graphs, new value in device memory
        want, margins = runs[p]
        got = dm.generate(ids, max_new_tokens=16, repetition_penalty=p).cpu()
        assert check_ids(got, want, margins, 12) >= 1, p
    neutral = dict(repetition_penalty=1.0, no_repeat_ngram_size=0, min_new_tokens=0)
    assert torch.equal(dm.generate(ids, max_new_tokens=16, **neutral).cpu(), greedy)
    assert torch.equal(dm.generate(ids, **sample_kw, **neutral).cpu(), sampled)
    assert torch.equal(dm.generate(ids, max_new_tokens=16).cpu(), greedy)


def test_sampling_with_processors_stays_in_hf_kept_set(models):
    cfg, dm, _ = models("TINY_QWEN2")
    ids = synthetic_tokens(cfg, 2, 12, seed=13)
    kw = dict(do_sample=True, temperature=0.9, top_k=20, top_p=0.95, max_new_tokens=16, repetition_penalty=1.3,
              no_repeat_ngram_size=2)
    a = dm.generate(ids, seed=11, **kw).cpu()
    assert torch.equal(a, dm.generate(ids, seed=11, **kw).cpu())
    assert not torch.equal(a, dm.generate(ids, seed=12, **kw).cpu())
    logits = dm(a[:, :-1]).logits.cpu()                            # teacher-forced logits of every prefix
    for r in range(2):
        for s in range(16):
            scores = hf_processed(logits[r:r + 1, 11 + s], [a[r, :12 + s]], 1.3, 2)
            # (prefill and decode logits differ in the last bf16 bit: a slightly wider set absorbs boundary flips)
            p = hf_warped(scores, 0.9, 24, 0.97)[0]
            assert float(p[a[r, 12 + s]]) > 0, (r, s)


def test_forward_still_refuses_the_keywords(models):
    cfg, dm, _ = models("TINY_QWEN2")
    ids = synthetic_tokens(cfg, 1, 4)
    with pytest.raises(NotImplementedError):
        dm(ids, repetition_penalty=1.2)
    with pytest.raises(ValueError):
        dm.generate(ids, max_new_tokens=2, repetition_penalty=0.0)
    assert M._logits_processors(1.0, 0, 0) is None
