"""The score log of ``generate(return_dict_in_generate=True, output_scores=True, output_logits=True)``.

Kernel level: each ``_log`` entry point against the same call without the log (ids, counters and histories bit for bit
unchanged), the raw log against ``logits.float()``, the processed log against HF's processors, the sampled log against
the sampler's own kept set (tests/rowwise_cases.py ``sample_row_model``) and, on pinned rows, HF's warpers; sentinels
around the written block and the column counter, eagerly and over graph replays.
End to end on tiny models: sequences equal plain generate's, scores against HF's rules on the logged logits, logits
against HF's own generate, graph == eager, micro-batches, left padding, EOS, FP8, and one full-size Qwen2.5-0.5B run."""
import numpy as np
import pytest
import torch

from tensorlink_b200.ml import configs as C
from tensorlink_b200.ml.weights import init_state_dict, synthetic_tokens
from tests.rowwise_cases import sample_row_model
from tests.scores_ref import hf_processed, hf_warped_scores, kept_scores

pytestmark = pytest.mark.gpu

SENT = -12345.5                  # a value no log entry takes
OUT = dict(return_dict_in_generate=True, output_scores=True, output_logits=True)


@pytest.fixture(scope="module")
def nat():
    from tensorlink_b200 import native
    native.require_device()
    return native


@pytest.fixture(autouse=True)
def _release_memory():
    yield
    import gc
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------- kernel level
class Log:
    """Sentinel-filled logs [n_cols, B_total, V] and a column counter starting at ``col``."""

    def __init__(self, n_cols, B_total, V, col=1):
        self.raw = torch.full((n_cols, B_total, V), SENT, device="cuda")
        self.sc = torch.full((n_cols, B_total, V), SENT, device="cuda")
        self.col = torch.tensor([col, 0], dtype=torch.int32, device="cuda")

    def arg(self, row0):
        return (self.raw, self.sc, self.col, row0)

    def block(self, c, row0, M):
        """(raw, scores) of the written block, after checking that nothing else changed."""
        for t in (self.raw, self.sc):
            rest = t.clone()
            rest[c, row0:row0 + M] = SENT
            assert bool((rest == SENT).all()), "a log entry outside the written block changed"
        return self.raw[c, row0:row0 + M].cpu(), self.sc[c, row0:row0 + M].cpu()


class Hist:
    def __init__(self, nat, prompt, V):
        M, S = prompt.shape
        self.log = torch.zeros(M, S + 4, dtype=torch.int32, device="cuda")
        self.len = torch.zeros(M, dtype=torch.int32, device="cuda")
        self.bits = torch.zeros(M, (V + 31) // 32, dtype=torch.int32, device="cuda")
        nat.history_fill(prompt.cuda().contiguous(), self.log, self.len, self.bits, V)

    def state(self):
        return self.log.clone(), self.len.clone(), self.bits.clone()


MS = [1, 2, 3, 4, 5, 6, 7, 8, 32]
VS = [1000, 32000, 151936, 152064]
PROC = dict(penalty=1.3, ngram=2, min_new=3)
WARP = dict(temperature=0.7, top_k=50, top_p=0.9)
WARP_PROC = dict(temperature=1.3, top_k=0, top_p=0.8)


def _case(M, V):
    g = torch.Generator().manual_seed(M * 7 + V)
    logits = (torch.randn(M, V, generator=g) * 2.5).bfloat16()
    S = 24
    pool = torch.randint(0, V, (M, 6), generator=g)
    prompt = torch.gather(pool, 1, torch.randint(0, 6, (M, S), generator=g))      # repeats: n-gram bans, penalties
    logits[:, pool[:, 0]] = 9.0                        # a penalised token near the top
    eos = (int(pool[0, 1]), 3)
    return logits, prompt, eos


def _run(nat, kind, logits_d, prompt, eos, log):
    """One call of ``kind`` with fresh counters and history; returns (ids, counters, history state)."""
    M, V = logits_d.shape
    ids = torch.full((M,), -1, dtype=torch.int64, device="cuda")
    ctr = torch.arange(M, dtype=torch.int32, device="cuda") * 3
    h = Hist(nat, prompt, V)
    if kind == "argmax":
        ws = torch.empty(M * 64 * 8 + 256, dtype=torch.uint8, device="cuda")
        nat.argmax_bf16(logits_d, ids, ws, log=log)
    elif kind == "sample":
        nat.sample(logits_d, ids, ctr, torch.empty(nat.sample_ws(M), dtype=torch.uint8, device="cuda"), seed=77, log=log, **WARP)
    else:
        ws = torch.empty(nat.logits_proc_ws(M, V), dtype=torch.uint8, device="cuda")
        params = nat.lp_params(PROC["penalty"], PROC["ngram"], PROC["min_new"], prompt.shape[1], eos).cuda()
        flags = nat.LP_BAN
        if kind == "argmax_proc":
            nat.argmax_proc(logits_d, ids, h.log, h.len, h.bits, params, ws, flags, score_log=log)
        else:
            nat.sample_proc(logits_d, ids, h.log, h.len, h.bits, params, ctr, ws, seed=77, flags=flags, score_log=log,
                            **WARP_PROC)
    return ids.cpu(), ctr.cpu(), [t.cpu() for t in h.state()]


def _hf_banned_rows(logits, prompt, eos):
    """HF's processed rows (history = prompt, min_new_tokens counted from the prompt's end) and per row (present, banned)."""
    M, V = logits.shape
    hist = [prompt[m] for m in range(M)]
    proc = hf_processed(logits, hist, PROC["penalty"], PROC["ngram"], PROC["min_new"], prompt.shape[1], eos)
    pen = hf_processed(logits, hist, PROC["penalty"])
    rows = []
    for m in range(M):
        present = np.zeros(V, bool)
        present[prompt[m].numpy()] = True
        rows.append((present, (proc[m] == float("-inf")).numpy() & (pen[m] != float("-inf")).numpy()))
    return proc, rows


def _check_kept_set(m, got_row, rm, x, T, what):
    kept = torch.from_numpy(rm.kept) if not rm.banned_all else torch.zeros_like(x, dtype=torch.bool)
    want = kept_scores(x.view(1, -1), kept.view(1, -1), T)[0]
    assert torch.equal(got_row, want), (what, m, int((got_row != want).sum()))


@pytest.mark.parametrize("V", VS)
@pytest.mark.parametrize("M", MS)
@pytest.mark.parametrize("kind", ["argmax", "argmax_proc", "sample", "sample_proc"])
def test_log_entry_points(nat, kind, M, V):
    logits, prompt, eos = _case(M, V)
    ld = logits.cuda()
    plain = _run(nat, kind, ld, prompt, eos, None)
    lg = Log(3, M + 2, V)
    logged = _run(nat, kind, ld, prompt, eos, lg.arg(1))
    assert torch.equal(plain[0], logged[0]) and torch.equal(plain[1], logged[1])        # ids, counters
    assert all(torch.equal(a, b) for a, b in zip(plain[2], logged[2]))                    # history
    assert lg.col.cpu().tolist() == [2, 0]                                                # one column; exit word back to 0
    raw, sc = lg.block(1, 1, M)
    assert torch.equal(raw, logits.float())
    ids = logged[0]
    if kind == "argmax":
        assert torch.equal(sc, logits.float())
        assert torch.equal(sc.argmax(-1), ids)
        return
    if kind == "argmax_proc":
        proc, _ = _hf_banned_rows(logits, prompt, eos)
        assert torch.equal(sc, proc)
        return
    if kind == "sample":
        T = WARP["temperature"]
        for m in range(M):
            rm = sample_row_model(logits[m], T, WARP["top_k"], WARP["top_p"])
            _check_kept_set(m, sc[m], rm, logits[m].float(), T, kind)
            assert torch.isfinite(sc[m, ids[m]])
            if rm.pinned:
                hf = hf_warped_scores(logits[m:m + 1].float(), T, WARP["top_k"], WARP["top_p"])[0]
                diff = torch.isfinite(hf) != torch.isfinite(sc[m])
                # HF's sort may split a group of equal values at the top-p boundary; the sampler keeps the whole group
                assert bool((logits[m].float()[diff] == logits[m].float()[torch.isfinite(sc[m])].min()).all()), m
        return
    T = WARP_PROC["temperature"]
    proc, rows = _hf_banned_rows(logits, prompt, eos)
    for m in range(M):
        present, banned = rows[m]
        rm = sample_row_model(logits[m], T, WARP_PROC["top_k"], WARP_PROC["top_p"], proc=True, present=present,
                              banned=banned, penalty=PROC["penalty"])
        _check_kept_set(m, sc[m], rm, proc[m], T, kind)
        if rm.banned_all:
            assert int(ids[m]) == 0 and bool((sc[m] == float("-inf")).all())
            continue
        assert torch.isfinite(sc[m, ids[m]])
        if rm.pinned:
            hf = hf_warped_scores(proc[m:m + 1], T, 0, WARP_PROC["top_p"])[0]
            diff = torch.isfinite(hf) != torch.isfinite(sc[m])
            assert bool((proc[m][diff] == proc[m][torch.isfinite(sc[m])].min()).all()), m


def test_every_token_banned(nat):
    """n = 1 over a history holding every id: the argmax logs -inf scores and picks 0; the sampler logs -inf everywhere."""
    V = 1000
    prompt = torch.arange(V, dtype=torch.int64).flip(0).view(1, V)
    logits = torch.randn(1, V, generator=torch.Generator().manual_seed(1)).bfloat16()
    ws = torch.empty(nat.logits_proc_ws(1, V), dtype=torch.uint8, device="cuda")
    params = nat.lp_params(1.0, 1, 0, V, []).cuda()
    for kind in ("argmax", "sample"):
        h = Hist(nat, prompt, V)
        lg = Log(1, 1, V, col=0)
        ids = torch.full((1,), 7, dtype=torch.int64, device="cuda")
        if kind == "argmax":
            nat.argmax_proc(logits.cuda(), ids, h.log, h.len, h.bits, params, ws, nat.LP_BAN, score_log=lg.arg(0))
        else:
            ctr = torch.zeros(1, dtype=torch.int32, device="cuda")
            nat.sample_proc(logits.cuda(), ids, h.log, h.len, h.bits, params, ctr, ws, 0.9, 0, 0.9, 3, nat.LP_BAN,
                            score_log=lg.arg(0))
        raw, sc = lg.block(0, 0, 1)
        assert int(ids) == 0 and lg.col.cpu().tolist() == [1, 0], kind
        assert torch.equal(raw, logits.float()) and bool((sc == float("-inf")).all()), kind
        assert torch.equal(sc, hf_processed(logits, [prompt[0]], 1.0, 1)), kind


def test_only_one_kind_and_column_guard(nat):
    M, V = 3, 1000
    logits, _, _ = _case(M, V)
    ld = logits.cuda()
    ids = torch.empty(M, dtype=torch.int64, device="cuda")
    ws = torch.empty(M * 64 * 8 + 256, dtype=torch.uint8, device="cuda")
    lg = Log(2, M, V, col=0)
    nat.argmax_bf16(ld, ids, ws, log=(lg.raw, None, lg.col, 0))
    assert torch.equal(lg.raw[0].cpu(), logits.float()) and bool((lg.sc == SENT).all())
    nat.argmax_bf16(ld, ids, ws, log=(None, lg.sc, lg.col, 0))
    assert torch.equal(lg.sc[1].cpu(), logits.float())
    before = (lg.raw.clone(), lg.sc.clone())
    nat.argmax_bf16(ld, ids, ws, log=lg.arg(0))          # column 2 of a 2-column log: not written, still advanced
    assert torch.equal(lg.raw, before[0]) and torch.equal(lg.sc, before[1])
    assert lg.col.cpu().tolist() == [3, 0]


@pytest.mark.parametrize("kind", ["argmax", "sample"])
def test_graph_replays_advance_one_column_each(nat, kind):
    M, V, n = 4, 32000, 100
    logits, prompt, eos = _case(M, V)
    ld = logits.cuda()
    lg = Log(n + 2, M, V, col=0)
    ids = torch.empty(M, dtype=torch.int64, device="cuda")
    ctr = torch.zeros(M, dtype=torch.int32, device="cuda")
    sws = torch.empty(nat.sample_ws(M), dtype=torch.uint8, device="cuda")
    aws = torch.empty(M * 64 * 8 + 256, dtype=torch.uint8, device="cuda")

    def step():
        if kind == "argmax":
            nat.argmax_bf16(ld, ids, aws, log=lg.arg(0))
        else:
            nat.sample(ld, ids, ctr, sws, seed=3, log=lg.arg(0), **WARP)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()                                           # warm-up: column 0
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    for _ in range(n):
        g.replay()
    torch.cuda.synchronize()
    assert lg.col.cpu().tolist() == [n + 1, 0]
    raw = lg.raw.cpu()
    for c in range(n + 1):
        assert torch.equal(raw[c], logits.float()), c
    assert bool((raw[n + 1] == SENT).all())


# ---------------------------------------------------------------------------------------------------- end to end
@pytest.fixture(scope="module")
def models():
    from tensorlink_b200.ml import DistributedModel
    cache = {}

    def get(name, max_batch=12, n_pipelines=1):
        key = (name, max_batch, n_pipelines)
        if key not in cache:
            cache[key] = DistributedModel(getattr(C, name), training=False, max_batch=max_batch, max_seq=256,
                                          n_pipelines=n_pipelines)
        return getattr(C, name), cache[key]
    return get


PROC_SETS = {"penalty": dict(repetition_penalty=1.3), "ngram": dict(no_repeat_ngram_size=2),
             "all": dict(repetition_penalty=1.2, no_repeat_ngram_size=3, min_new_tokens=4)}
SAMPLE = dict(do_sample=True, temperature=0.8, top_k=40, top_p=0.9, seed=21)
MODES = ["greedy", "sampled"] + list(PROC_SETS) + [f"sampled_{p}" for p in PROC_SETS]


def _mode_kw(mode):
    kw = dict(SAMPLE) if mode.startswith("sampled") else {}
    p = mode.replace("sampled", "").replace("greedy", "").strip("_")
    if p:
        kw.update(PROC_SETS[p])
    return kw


def _check_scores(o, S, kw):
    """scores against HF's rules applied to the logged logits, column by column."""
    seq = o.sequences.cpu()
    T = len(o.scores)
    assert T == len(o.logits) == seq.shape[1] - S
    B = seq.shape[0]
    penalty = kw.get("repetition_penalty", 1.0)
    ngram = kw.get("no_repeat_ngram_size", 0)
    min_new = kw.get("min_new_tokens", 0)
    for c in range(T):
        sc, lo = o.scores[c].cpu(), o.logits[c].cpu()
        assert sc.shape == lo.shape == (B, lo.shape[1]) and sc.dtype == lo.dtype == torch.float32
        assert torch.equal(lo.bfloat16().float(), lo)                       # float(bf16 logit)
        proc = hf_processed(lo.bfloat16(), [seq[r, :S + c] for r in range(B)], penalty, ngram, min_new, S, ())
        tok = seq[:, S + c]
        if "do_sample" in kw:
            assert bool(torch.isfinite(sc[torch.arange(B), tok]).all()), c
            fin = torch.isfinite(sc)
            assert torch.equal(sc[fin], (proc / torch.tensor(kw["temperature"]))[fin]), c
        else:
            assert torch.equal(sc, proc), c
            assert torch.equal(sc.argmax(-1), tok), c


@pytest.mark.parametrize("name", ["TINY_QWEN2", "TINY_QWEN3"])
@pytest.mark.parametrize("B", [1, 3, 12])
@pytest.mark.parametrize("mode", MODES)
def test_generate_scores(models, name, B, mode):
    cfg, dm = models(name)
    kw = _mode_kw(mode)
    ids = synthetic_tokens(cfg, B, 10, seed=B)
    plain = dm.generate(ids, max_new_tokens=16, **kw).cpu()
    o = dm.generate(ids, max_new_tokens=16, output_scores=True, output_logits=True, return_dict_in_generate=True, **kw)
    assert torch.equal(o.sequences.cpu(), plain)
    assert o.attentions is None and o.hidden_states is None and o.past_key_values is None
    assert o.scores[0].device == o.sequences.device
    _check_scores(o, 10, kw)
    if B == 3:
        e = dm.generate(ids, max_new_tokens=16, use_graph=False, **OUT, **kw)
        assert torch.equal(e.sequences, o.sequences)
        assert all(torch.equal(a, b) for a, b in zip(e.scores, o.scores))
        assert all(torch.equal(a, b) for a, b in zip(e.logits, o.logits))
    # only one kind asked for: the other is None, the asked one unchanged
    s = dm.generate(ids, max_new_tokens=16, output_scores=True, return_dict_in_generate=True, **kw)
    assert s.logits is None and all(torch.equal(a, b) for a, b in zip(s.scores, o.scores))
    g = dm.generate(ids, max_new_tokens=16, output_logits=True, return_dict_in_generate=True, **kw)
    assert g.scores is None and all(torch.equal(a, b) for a, b in zip(g.logits, o.logits))


@pytest.mark.parametrize("name", ["TINY_QWEN2", "TINY_QWEN3"])
def test_logits_agree_with_hf_generate(models, name):
    """HF's own generate on the same weights: the logits agree within bf16 tolerance at every column up to the first
    column where the two token sequences part."""
    from tests.hf_util import hf_model
    MARGIN = 0.05
    cfg, dm = models(name)
    hf = hf_model(cfg, init_state_dict(cfg))
    hf.generation_config.eos_token_id = None
    hf.generation_config.pad_token_id = 0
    checked = 0
    for seed in range(3, 43):
        ids = synthetic_tokens(cfg, 3, 10, seed=seed)
        want = hf.generate(ids, attention_mask=torch.ones_like(ids), max_new_tokens=12, do_sample=False, output_scores=True,
                           output_logits=True, return_dict_in_generate=True)
        top2 = torch.stack(want.logits, 1).float().topk(2, -1).values
        if not bool((top2[:, 0, 0] - top2[:, 0, 1] >= MARGIN).any()):
            continue
        got = dm.generate(ids, max_new_tokens=12, **OUT)
        gs, ws = got.sequences.cpu(), want.sequences
        for c in range(12):
            a, b = got.logits[c].cpu(), want.logits[c].float()
            scale = float(b.abs().max())
            assert float((a - b).abs().max()) <= 2 ** -5 * scale + 2 ** -6, (c, float((a - b).abs().max()), scale)
            checked += 1
            if not torch.equal(gs[:, 10 + c], ws[:, 10 + c]):
                break
        break
    assert checked >= 1


def test_micro_batches_equal_halves(models):
    cfg, one = models("TINY_QWEN2", 2, 1)
    _, two = models("TINY_QWEN2", 4, 2)
    ids = synthetic_tokens(cfg, 4, 9, seed=3)
    for kw in (dict(repetition_penalty=1.3), SAMPLE):
        both = two.generate(ids, max_new_tokens=12, **OUT, **kw)
        for h in range(2):
            # slot h draws with the key seed + GOLDEN * h (ml/stage.py): the one-slot run of half h takes that key
            kh = dict(kw, seed=(kw["seed"] + 0x9E3779B97F4A7C15 * h) % 2 ** 64) if "do_sample" in kw else kw
            half = one.generate(ids[2 * h:2 * h + 2], max_new_tokens=12, **OUT, **kh)
            assert torch.equal(both.sequences[2 * h:2 * h + 2], half.sequences), (kw, h)
            for c in range(12):
                assert torch.equal(both.scores[c][2 * h:2 * h + 2], half.scores[c]), (kw, h, c)
                assert torch.equal(both.logits[c][2 * h:2 * h + 2], half.logits[c]), (kw, h, c)


def test_left_padded_batch(models):
    cfg, dm = models("TINY_QWEN2")
    lengths = (6, 11, 8)
    S = max(lengths) + 1
    ids = torch.full((3, S), 5, dtype=torch.int64)
    mask = torch.zeros(3, S, dtype=torch.int64)
    for b, L in enumerate(lengths):
        ids[b, S - L:], mask[b, S - L:] = synthetic_tokens(cfg, 1, L, seed=10 * b)[0], 1
    plain = dm.generate(ids, attention_mask=mask, max_new_tokens=10).cpu()
    o = dm.generate(ids, attention_mask=mask, max_new_tokens=10, **OUT)
    assert torch.equal(o.sequences.cpu(), plain)
    _check_scores(o, S, {})
    p = dm.generate(ids, attention_mask=mask, max_new_tokens=10, repetition_penalty=1.5, **OUT)
    _check_scores(p, S, dict(repetition_penalty=1.5))                   # the pad columns count as seen, as in HF


def test_eos_cuts_the_columns(models):
    cfg, dm = models("TINY_QWEN3")
    ids = synthetic_tokens(cfg, 3, 10, seed=4)
    full = dm.generate(ids, max_new_tokens=40, **OUT)
    eos = int(full.sequences[0, 10 + 1])
    o = dm.generate(ids, max_new_tokens=40, eos_token_id=eos, pad_token_id=0, **OUT)
    seq = o.sequences.cpu()
    assert torch.equal(seq, dm.generate(ids, max_new_tokens=40, eos_token_id=eos, pad_token_id=0).cpu())
    assert len(o.scores) == len(o.logits) == seq.shape[1] - 10
    one = dm.generate(ids[:1], max_new_tokens=40, eos_token_id=eos, pad_token_id=0, **OUT)
    assert one.sequences.shape[1] == 12 and len(one.scores) == len(one.logits) == 2     # 14 surplus columns dropped
    for r in range(3):
        new = seq[r, 10:].tolist()
        end = new.index(eos) + 1 if eos in new else len(new)
        for c in range(end):                                       # up to its EOS a row's columns are its own decode's
            assert int(o.scores[c][r].argmax()) == new[c], (r, c)
            assert torch.equal(o.scores[c][r], full.scores[c][r])


def test_one_new_token_and_no_aliasing(models):
    cfg, dm = models("TINY_QWEN2")
    ids = synthetic_tokens(cfg, 2, 8, seed=1)
    one = dm.generate(ids, max_new_tokens=1, **OUT)
    assert len(one.scores) == len(one.logits) == 1 and one.sequences.shape[1] == 9
    a = dm.generate(ids, max_new_tokens=6, **OUT)
    keep = [t.clone() for t in a.scores + a.logits]
    dm.generate(synthetic_tokens(cfg, 2, 8, seed=2), max_new_tokens=6, **OUT)
    assert all(torch.equal(x, y) for x, y in zip(a.scores + a.logits, keep))


def test_plain_call_keeps_its_graph_launches(models):
    """After a logging call the plain call captures its own graphs again: the log is off and its tokens unchanged."""
    cfg, dm = models("TINY_QWEN2")
    ids = synthetic_tokens(cfg, 2, 8, seed=6)
    before = dm.generate(ids, max_new_tokens=8).cpu()
    dm.generate(ids, max_new_tokens=8, **OUT)
    assert dm.stage.log_mode == (True, True)
    assert torch.equal(dm.generate(ids, max_new_tokens=8, output_scores=True).cpu(), before)
    assert dm.stage.log_mode == (False, False)
    assert all(k[3] == (False, False) for k in dm.stage.graphs)


def test_fp8_scores_equal_bf16_over_dequantized():
    from tests.test_fp8_gpu import _pair
    cfg = C.TINY_QWEN2
    f, b, _ = _pair(cfg, max_batch=8)
    for B, kw in ((1, {}), (3, SAMPLE), (8, dict(repetition_penalty=1.3))):
        ids = synthetic_tokens(cfg, B, 10, seed=B)
        x, y = f.generate(ids, max_new_tokens=12, **OUT, **kw), b.generate(ids, max_new_tokens=12, **OUT, **kw)
        assert torch.equal(x.sequences, y.sequences)
        assert all(torch.equal(p, q) for p, q in zip(x.scores + x.logits, y.scores + y.logits)), B


def test_full_size_qwen25_05b():
    from oracle import shard_oracle as O
    from tensorlink_b200.ml import DistributedModel
    cfg = C.QWEN25_05B
    sd = init_state_dict(cfg)
    ids = synthetic_tokens(cfg, 1, 32)
    dm = DistributedModel(cfg, training=False, max_batch=1, max_seq=128)
    plain = dm.generate(ids, max_new_tokens=16).cpu()
    o = dm.generate(ids, max_new_tokens=16, **OUT)
    assert torch.equal(o.sequences.cpu(), plain)
    _check_scores(o, 32, {})
    with torch.no_grad():
        ref16 = O.OracleModel(cfg, sd, "sdpa_math").logits(ids)[:, -1].float()
        ref32 = O.OracleModel(cfg, {k: v.float() for k, v in sd.items()}, "sdpa_math").logits(ids)[:, -1].float()
    err, floor = O.rel_l2(o.logits[0].cpu(), ref32), O.rel_l2(ref16, ref32)
    assert err <= 2 * floor + 1e-3, (err, floor)
