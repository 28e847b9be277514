"""Prompt-lookup decoding on the GPU: the draft and accept kernels (csrc/prompt_lookup.cu), the verify attention
(attention.cu), the stage's verify step and ``generate(prompt_lookup_num_tokens=K)``.

  * draft kernel: candidate for candidate against HF's PromptLookupCandidateGenerator.get_candidates;
  * accept kernel: exact, on crafted inputs, including what must not move;
  * verify attention: row by row against float64 with the criteria of tests/test_attention_numerics_gpu.py, with the
    cache above the last query's slot poisoned (NaN, then huge finite values);
  * verify step and generate: greedy ids against the CPU oracle wherever its top-2 margin is resolvable (MARGIN), as
    in tests/test_model_gpu.py, and graph replay against eager launches bit for bit.
"""
import random

import pytest
import torch

from oracle import shard_oracle as O
from tensorlink_b200.ml import configs as C
from tensorlink_b200.ml.module import apply_eos
from tensorlink_b200.ml.weights import init_state_dict, synthetic_tokens
from tests import attn_patterns as P
from tests.test_attention_numerics_gpu import FWD_FLOOR, FWD_K, check_rows, oracle_fwd, ref_fwd

pytestmark = pytest.mark.gpu
MARGIN = 0.05
SENTINEL = 999_999


@pytest.fixture(scope="module")
def nat():
    from tensorlink_b200 import native
    native.require_device()
    return native


# ------------------------------------------------------------------------------------------ draft kernel vs HF
def _hf_candidates(hist, K, n, max_length, eos):
    from transformers.generation.candidate_generator import PromptLookupCandidateGenerator
    gen = PromptLookupCandidateGenerator(eos_token_id=torch.tensor(eos, dtype=torch.int64), num_output_tokens=K,
                                         max_matching_ngram_size=n, max_length=max_length)
    ids = torch.tensor([hist], dtype=torch.int64)
    out, _ = gen.get_candidates(ids)
    return out[0, len(hist):].tolist()


def _draft(nat, hist, K, n, max_length, eos, L_cap=512):
    log = torch.full((L_cap,), SENTINEL, dtype=torch.int32, device="cuda")      # past the length: never a candidate
    log[:len(hist)] = torch.tensor(hist, dtype=torch.int32)
    length = torch.tensor([len(hist)], dtype=torch.int32, device="cuda")
    params = nat.pl_params(n, max_length, eos).cuda()
    in_ids = torch.full((16,), -5, dtype=torch.int64, device="cuda")
    n_cand = torch.full((1,), -5, dtype=torch.int32, device="cuda")
    nat.pl_draft(log, length, params, K, in_ids, n_cand)
    c = int(n_cand.item())
    got = in_ids.cpu().tolist()
    assert got[0] == hist[-1] and all(t == hist[-1] for t in got[1 + c:K + 1]) and all(t == -5 for t in got[K + 1:])
    return got[1:1 + c]


@pytest.mark.parametrize("K", [1, 4, 10, 15])
@pytest.mark.parametrize("n", [1, 2, 3, 5])
def test_draft_matches_hf(nat, n, K):
    rng = random.Random(1000 * n + K)
    cases = 0
    for trial in range(80):
        L = rng.choice([1, 2, 3, 4, 5, 8, 17, 40, 100, 257, 300])
        vocab = rng.choice([2, 3, 5])                       # tiny vocabularies: matches everywhere
        hist = [rng.randrange(vocab) for _ in range(L)]
        eos = rng.choice([[], [rng.randrange(vocab)], [0, 1]])
        max_length = rng.choice([L + 1, L + 2, L + 3, L + 500])
        want = _hf_candidates(hist, K, n, max_length, eos)
        got = _draft(nat, hist, K, n, max_length, eos)
        assert got == want, (trial, L, hist[-8:], eos, max_length, got, want)
        cases += bool(want)
    assert cases >= 20                                      # most histories do give candidates


def test_draft_eos_first_candidate(nat):
    hist = [1, 2, 7, 3, 4, 5, 1, 2]                         # "1 2" recurs; it was followed by 7
    assert _draft(nat, hist, 4, 2, 100, []) == [7, 3, 4, 5] == _hf_candidates(hist, 4, 2, 100, [])
    assert _draft(nat, hist, 4, 2, 100, [7]) == [] == _hf_candidates(hist, 4, 2, 100, [7])
    assert _draft(nat, hist, 4, 2, 100, [9, 4]) == [7, 3] == _hf_candidates(hist, 4, 2, 100, [9, 4])
    assert _draft(nat, hist, 4, 2, len(hist) + 1, []) == []                       # max_length == L + 1
    assert _draft(nat, hist, 4, 2, len(hist) + 2, []) == [7, 3, 4, 5]


# ------------------------------------------------------------------------------------------ accept kernel
def _accept(nat, in_ids, ids, n_cand, K, length=20, count=3, pos=19, max_length=40, L_cap=64, V=100):
    dev = "cuda"
    log = torch.full((L_cap,), -1, dtype=torch.int32, device=dev)
    log[:length] = torch.arange(length, dtype=torch.int32)
    bits = torch.zeros((V + 31) // 32, dtype=torch.int32, device=dev)
    st = {"log": log, "len": torch.tensor([length], dtype=torch.int32, device=dev), "bits": bits,
          "out": torch.full((32,), -7, dtype=torch.int64, device=dev),
          "count": torch.tensor([count], dtype=torch.int32, device=dev),
          "pos": torch.tensor([pos], dtype=torch.int32, device=dev), "kvl": torch.tensor([pos - 3], dtype=torch.int32, device=dev)}
    ids_t = torch.full((16,), 55, dtype=torch.int64, device=dev)
    ids_t[:K + 1] = torch.tensor(ids)
    in_t = torch.full((16,), 66, dtype=torch.int64, device=dev)
    in_t[:K + 1] = torch.tensor(in_ids)
    nc = torch.tensor([n_cand], dtype=torch.int32, device=dev)
    params = nat.pl_params(2, max_length, []).cuda()
    nat.pl_accept(ids_t, in_t, nc, st["log"], st["len"], st["bits"], V, params, st["out"], st["count"], st["pos"], st["kvl"], K)
    return {k: v.cpu() for k, v in st.items()}


def _check_accept(st, emitted, length=20, count=3, pos=19, V=100):
    e = len(emitted)
    assert int(st["len"]) == length + e and int(st["count"]) == count + e
    assert int(st["pos"]) == pos + e and int(st["kvl"]) == pos + e
    assert st["log"][:length].tolist() == list(range(length))
    assert st["log"][length:length + e].tolist() == emitted and bool((st["log"][length + e:] == -1).all())
    assert bool((st["out"][:count] == -7).all()) and st["out"][count:count + e].tolist() == emitted
    assert bool((st["out"][count + e:] == -7).all())
    want_bits = torch.zeros((V + 31) // 32, dtype=torch.int64)
    for t in emitted:
        want_bits[t >> 5] |= 1 << (t & 31)
    assert torch.equal(st["bits"].to(torch.int64) & 0xFFFFFFFF, want_bits)


def test_accept_exact(nat):
    K = 5
    x, c = 10, [11, 12, 13, 14, 15]
    ins = [x] + c
    # all accepted: the model agrees with every draft and adds its own next token
    _check_accept(_accept(nat, ins, [11, 12, 13, 14, 15, 16], 5, K), [11, 12, 13, 14, 15, 16])
    # none accepted
    _check_accept(_accept(nat, ins, [40, 12, 13, 14, 15, 16], 5, K), [40])
    # first mismatch at each i
    for i in range(K):
        ids = [11, 12, 13, 14, 15, 16]
        ids[i] = 41
        _check_accept(_accept(nat, ins, ids, 5, K), [11, 12, 13, 14, 15, 16][:i] + [41])
    # n_cand < K: the filler row agrees with the model but is never accepted
    ins2 = [x, 11, 12, 77, 77, 77]
    _check_accept(_accept(nat, ins2, [11, 12, 77, 77, 77, 77], 2, K), [11, 12, 77])
    _check_accept(_accept(nat, ins2, [11, 12, 77, 77, 77, 77], 0, K), [11])
    # the max_new boundary: the history may grow by max_length - len tokens at most, and not at all once full
    _check_accept(_accept(nat, ins, [11, 12, 13, 14, 15, 16], 5, K, max_length=23), [11, 12, 13])
    _check_accept(_accept(nat, ins, [11, 12, 13, 14, 15, 16], 5, K, max_length=21), [11])
    _check_accept(_accept(nat, ins, [11, 12, 13, 14, 15, 16], 5, K, max_length=20), [])


# ------------------------------------------------------------------------------------------ verify attention
LAYOUTS = [(4, 4, 64), (4, 2, 64), (4, 2, 128), (32, 8, 128), (14, 2, 64), (28, 4, 128), (16, 2, 128)]   # n_rep 1..8


@pytest.mark.parametrize("n_h,n_kv,d", LAYOUTS)
@pytest.mark.parametrize("q_len", [1, 2, 3, 4, 8, 11, 16])
def test_verify_attention_vs_float64(nat, q_len, n_h, n_kv, d):
    scale = d ** -0.5
    for pos, pattern in ((37, "flat"), (250, "rising"), (256, "spike@255"), (256 - q_len // 2, "spike@256"),
                         (2900, "wide")):
        T = pos + q_len
        T_max = T + 100
        q, k = P.make_qk(pattern, 1, q_len, T, n_h, n_kv, d, seed=pos + q_len)
        v = P.make_v(1, n_kv, T, d, seed=pos + 7)
        q, k, v = q.cuda(), k.cuda(), v.cuda()
        ref, _ = ref_fwd(q, k, v, pos, scale)
        orc = oracle_fwd(q, k, v, scale)
        ws = torch.empty(nat.attn_verify_ws(q_len, n_h, d, T_max), dtype=torch.uint8, device="cuda")
        posd = torch.tensor([pos], dtype=torch.int32, device="cuda")
        outs = []
        for poison in (float("nan"), 1e30):
            kc = torch.full((1, n_kv, T_max, d), poison, dtype=torch.bfloat16, device="cuda")
            vc = torch.full_like(kc, poison)
            kc[:, :, :T], vc[:, :, :T] = k, v
            out = torch.full((q_len, n_h * d), float("nan"), dtype=torch.bfloat16, device="cuda")
            nat.attn_verify_fwd(q.reshape(q_len, n_h * d), kc, vc, out, posd, ws, q_len, n_h, n_kv, d, scale)
            check_rows(f"verify q_len={q_len} pos={pos} {pattern} poison={poison}", out.view(1, q_len, n_h, d), ref, orc,
                       FWD_K, FWD_FLOOR)
            outs.append(out)
        assert torch.equal(outs[0], outs[1])               # what lies above the last query's slot never matters
        if q_len == 1:                                     # the decode kernel meets the same bound on the same rows
            dws = torch.empty(nat.attn_decode_ws(1, n_h, d, T_max), dtype=torch.uint8, device="cuda")
            dout = torch.empty(1, n_h * d, dtype=torch.bfloat16, device="cuda")
            nat.attn_decode_fwd(q.reshape(1, n_h * d), kc, vc, dout, torch.tensor([T], dtype=torch.int32, device="cuda"),
                                dws, 1, n_h, n_kv, d, scale)
            check_rows("decode q_len=1", dout.view(1, 1, n_h, d), ref, orc, FWD_K, FWD_FLOOR)


# ------------------------------------------------------------------------------------------ stage-level verify step
CASES = [C.TINY_QWEN2, C.TINY_QWEN2_D128, C.TINY_QWEN3]


def _make(cfg, **kw):
    from tensorlink_b200.ml import DistributedModel
    kw.setdefault("max_seq", 256)
    kw.setdefault("max_batch", 1)
    return DistributedModel(cfg, training=False, **kw)


def _begin(dm, ids, K, max_new):
    """What generate does before its first verify step."""
    st = dm.stage
    st.set_sampling(None)
    st.set_logits_processors(None)
    x = st.prefill(st.embed(ids.cuda()), 0, 0)
    first = st.ids_dec[0][:1]
    st.head_argmax(x[:, -1, :].contiguous(), first, 0)
    st.prompt_lookup_begin(torch.cat([ids.cuda(), first.view(1, 1)], dim=1), K, 2, ids.shape[1] + max_new, [])
    return int(first.item())


def _reliable(margins):
    """Steps 0..n-1 of the oracle's greedy run have a resolvable margin."""
    m = margins[0]
    bad = (m < MARGIN).nonzero()
    return int(bad[0]) if bad.numel() else m.numel()


@pytest.mark.parametrize("cfg", CASES, ids=lambda c: c.name)
@pytest.mark.parametrize("K", [2, 10])
def test_verify_step_given_drafts(cfg, K):
    sd = init_state_dict(cfg)
    oracle = O.OracleModel(cfg, sd, "sdpa_math")
    for S in (12, 10, 14, 9, 16, 11, 13):                   # the first prompt whose first steps the oracle resolves
        ids = synthetic_tokens(cfg, 1, S)
        ref, margins = oracle.generate(ids, K + 2, return_margins=True)
        n_ok = _reliable(margins)
        if n_ok >= 3:
            break
    assert n_ok >= 2, f"oracle margin below {MARGIN} at step {n_ok} for every prompt"
    want = ref[0, S:].tolist()
    dm = _make(cfg)
    assert _begin(dm, ids, K, 64) == want[0]
    drafts = want[1:K + 1]
    got = dm.stage.verify_drafts(drafts)
    n_cmp = min(len(got), n_ok - 1)
    assert got[:n_cmp] == want[1:1 + n_cmp], (got, want)
    assert len(got) - 1 >= min(K, n_ok - 1)                 # every resolvable draft is accepted
    print(f"{cfg.name} K={K}: {len(got) - 1} drafts accepted, oracle margins resolvable for {n_ok} steps")
    for j in range(min(K, n_ok - 1)):                       # a wrong draft at j: a = j, the model's token replaces it
        bad = list(drafts)
        bad[j] = (bad[j] + 1) % cfg.vocab
        _begin(dm, ids, K, 64)
        got = dm.stage.verify_drafts(bad)
        assert got == want[1:2 + j], (j, got, want)


# ------------------------------------------------------------------------------------------ generate
def _repeating_prompt(cfg, period=8, times=3):
    base = synthetic_tokens(cfg, 1, period)
    return base.repeat(1, times)


class _Streamer:
    def __init__(self):
        self.puts, self.ended = [], False

    def put(self, t):
        self.puts.append(t.clone())

    def end(self):
        self.ended = True


@pytest.mark.parametrize("cfg", CASES, ids=lambda c: c.name)
@pytest.mark.parametrize("K", [1, 3, 10])
def test_generate_prompt_lookup(cfg, K):
    from tests.test_model_gpu import _check_ids
    sd = init_state_dict(cfg)
    ids = _repeating_prompt(cfg)
    S, new = ids.shape[1], 40
    ref, margins = O.OracleModel(cfg, sd, "sdpa_math").generate(ids, new, return_margins=True)
    dm = _make(cfg)
    plain = dm.generate(ids, max_new_tokens=new).cpu()
    stream = _Streamer()
    got = dm.generate(ids, max_new_tokens=new, prompt_lookup_num_tokens=K, streamer=stream).cpu()
    steps = dm.timers["prompt_lookup_steps"]
    eager = dm.generate(ids, max_new_tokens=new, prompt_lookup_num_tokens=K, use_graph=False).cpu()
    again = dm.generate(ids, max_new_tokens=new).cpu()
    assert got.shape == (1, S + new) and torch.equal(got[:, :S], ids)
    assert torch.equal(got, eager)                          # CUDA-graph replay == eager launches, bit for bit
    assert torch.equal(plain, again)                        # the lookup run leaves plain decoding as it was
    # the oracle's greedy ids, and plain decoding, up to the first unresolvable step
    n = _check_ids(got, ref, margins, S)
    n_ok = _reliable(margins)
    assert torch.equal(got[:, S:S + n_ok], plain[:, S:S + n_ok])
    # teacher-forced: every token is the argmax of one forward over the final sequence where that margin is resolvable
    logits = dm(got[:, :-1]).logits[:, S - 1:].cpu().float()
    top2 = logits.topk(2, -1).values
    safe = (top2[..., 0] - top2[..., 1]) > MARGIN
    assert safe.float().mean() > 0.2
    assert torch.equal(logits.argmax(-1)[safe], got[:, S:][safe])
    # the streamer got every token once, in order
    assert stream.ended and all(t.numel() == 1 for t in stream.puts)
    assert torch.cat(stream.puts).tolist() == got[0, S:].tolist()
    print(f"{cfg.name} K={K}: {new} tokens in {steps} verify steps + the prefill's "
          f"({(new - 1) / max(steps, 1):.2f} tokens per step), {n} steps oracle-exact")
    assert steps < new - 1                                  # at least one draft was accepted
    # EOS: the lookup run stops where plain decoding does
    j = next((s for s in range(min(n_ok, new)) if got[0, S + s] not in got[0, S:S + s].tolist() and s >= 3), None)
    if j is not None:
        eos = int(got[0, S + j])
        p = dm.generate(ids, max_new_tokens=new, eos_token_id=eos).cpu()
        g = dm.generate(ids, max_new_tokens=new, eos_token_id=eos, prompt_lookup_num_tokens=K).cpu()
        assert torch.equal(g, p) and g.shape[1] == S + j + 1
        assert torch.equal(g, apply_eos(got, S, eos))


def test_generate_max_new_boundary():
    """Exactly max_new_tokens tokens for every max_new around a step of K+1, and one-token runs."""
    cfg = C.TINY_QWEN2
    dm = _make(cfg)
    ids = _repeating_prompt(cfg)
    S = ids.shape[1]
    full = dm.generate(ids, max_new_tokens=30, prompt_lookup_num_tokens=4).cpu()
    for m in (1, 2, 4, 5, 6, 11, 29):
        got = dm.generate(ids, max_new_tokens=m, prompt_lookup_num_tokens=4).cpu()
        assert got.shape == (1, S + m)
        assert dm.timers["prompt_lookup_steps"] <= m - 1
        assert torch.equal(got[:, :S + 1], full[:, :S + 1])


def test_full_size_qwen25_05b_k10():
    """Qwen2.5-0.5B at full size (device-initialised weights): K = 10 against plain decoding and against one forward
    over the final sequence, graph against eager."""
    cfg = C.QWEN25_05B
    dm = _make(cfg, max_seq=256, init="device")
    ids = synthetic_tokens(cfg, 1, 16).repeat(1, 4)
    S, new = ids.shape[1], 48
    plain = dm.generate(ids, max_new_tokens=new).cpu()
    got = dm.generate(ids, max_new_tokens=new, prompt_lookup_num_tokens=10).cpu()
    steps = dm.timers["prompt_lookup_steps"]
    eager = dm.generate(ids, max_new_tokens=new, prompt_lookup_num_tokens=10, use_graph=False).cpu()
    assert torch.equal(got, eager) and got.shape == plain.shape
    for seq in (plain, got):
        logits = dm(seq[:, :-1]).logits[:, S - 1:].cpu().float()
        top2 = logits.topk(2, -1).values
        safe = (top2[..., 0] - top2[..., 1]) > MARGIN
        assert safe.float().mean() > 0.2
        assert torch.equal(logits.argmax(-1)[safe], seq[:, S:][safe])
    diff = (got != plain)[0, S:].nonzero()
    print(f"Qwen2.5-0.5B K=10: {new} tokens in {steps} verify steps ({(new - 1) / max(steps, 1):.2f} tokens per step); "
          f"first divergence from plain decoding: {int(diff[0]) if diff.numel() else None}")
