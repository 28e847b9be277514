"""Assisted decoding on the GPU: ``generate(assistant_model=draft, num_assistant_tokens=K)``.

  * prep kernel (csrc/prompt_lookup.cu tl_assist_prep): exact on crafted histories, with sentinels around every buffer;
  * one round at a time (``CudaStage.verify_round``): the assistant's drafts against the CPU oracle's greedy continuation
    OF THE ASSISTANT over the sequence so far, the emitted tokens against the target oracle's, wherever the oracle's
    top-2 margin is resolvable (MARGIN) -- a misplaced or stale assistant cache slot changes the drafts;
  * generate on the tiny configs with three assistants (same weights: every draft accepted; another seed: almost every
    draft rejected; the target's first two layers: mixed acceptance) against the oracle, plain decoding, a
    teacher-forced forward, graph == eager and the streamer; mismatched vocabularies; max_new / EOS boundaries; the
    lifetime of the captured graphs; and a Qwen2.5-7B model with a Qwen2.5-0.5B assistant at full size.
"""
import functools

import pytest
import torch

from oracle import shard_oracle as O
from tensorlink_b200.ml import configs as C
from tensorlink_b200.ml.module import apply_eos
from tensorlink_b200.ml.weights import init_state_dict, synthetic_tokens

pytestmark = pytest.mark.gpu
MARGIN = 0.05
MARGIN_FULL = 0.25
SENTINEL = 999_999
CASES = [C.TINY_QWEN2, C.TINY_QWEN2_D128, C.TINY_QWEN3]
ASSISTANTS = ("same", "other_seed", "two_layers")


@pytest.fixture(scope="module")
def nat():
    from tensorlink_b200 import native
    native.require_device()
    return native


# ------------------------------------------------------------------------------------------ prep kernel
@pytest.mark.parametrize("L", [2, 3, 17, 64])
def test_prep_kernel_exact(nat, L):
    dev, L_cap, pad = "cuda", 64, 2
    hist = [(7 * i + 3) % 1000 for i in range(L)]

    def boxed(n, dtype, fill=SENTINEL):
        return torch.full((n + 2 * pad,), fill, dtype=dtype, device=dev)

    log_b = boxed(L_cap, torch.int32)
    log_b[pad:pad + L] = torch.tensor(hist, dtype=torch.int32)
    len_b = boxed(1, torch.int32)
    len_b[pad] = L
    asst_b, in_b = boxed(2, torch.int64), boxed(16, torch.int64)
    pos_b, kvl_b = boxed(1, torch.int32, -5), boxed(1, torch.int32, -6)
    before = [t.clone() for t in (log_b, len_b, asst_b, in_b, pos_b, kvl_b)]
    nat.assist_prep(log_b[pad:pad + L_cap], len_b[pad:pad + 1], asst_b[pad:pad + 2], in_b[pad:pad + 16],
                    pos_b[pad:pad + 1], kvl_b[pad:pad + 1])
    P = L - 1
    want = [t.clone() for t in before]
    want[2][pad:pad + 2] = torch.tensor([hist[P - 1], hist[P]])
    want[3][pad] = hist[P]
    want[4][pad] = P - 1
    want[5][pad] = P - 1
    for name, got, w in zip(("log", "len", "asst_in", "in_ids", "pos", "kv_len"), (log_b, len_b, asst_b, in_b, pos_b,
                                                                                   kvl_b), want):
        assert torch.equal(got, w), (name, got.cpu().tolist(), w.cpu().tolist())


# ------------------------------------------------------------------------------------------ models
def _make(cfg, seed=1234, **kw):
    from tensorlink_b200.ml import DistributedModel
    kw.setdefault("max_seq", 256)
    kw.setdefault("max_batch", 1)
    return DistributedModel(cfg, training=False, seed=seed, **kw)


def _assistant_cfg(cfg, kind):
    return cfg.scaled(n_layers=2) if kind == "two_layers" else cfg


def _assistant_seed(kind):
    return 99 if kind == "other_seed" else 1234


@functools.lru_cache(maxsize=None)
def _target(cfg):
    return _make(cfg)


@functools.lru_cache(maxsize=None)
def _assistant(cfg, kind):
    return _make(_assistant_cfg(cfg, kind), seed=_assistant_seed(kind))


@functools.lru_cache(maxsize=None)
def _oracle(cfg, seed=1234):
    return O.OracleModel(cfg, init_state_dict(cfg, seed), "sdpa_math")


def _reliable(margins):
    """Steps 0..n-1 of the oracle's greedy run have a resolvable margin."""
    m = margins[0]
    bad = (m < MARGIN).nonzero()
    return int(bad[0]) if bad.numel() else m.numel()


@functools.lru_cache(maxsize=None)
def _prompt(cfg):
    """The first synthetic prompt whose first greedy steps the oracle resolves."""
    for S in (12, 10, 14, 9, 16, 11, 13):
        ids = synthetic_tokens(cfg, 1, S)
        if _reliable(_oracle(cfg).generate(ids, 6, return_margins=True)[1]) >= 4:
            return ids
    raise AssertionError(f"oracle margin below {MARGIN} within 4 steps for every prompt")


# ------------------------------------------------------------------------------------------ one round at a time
@pytest.mark.parametrize("cfg", CASES, ids=lambda c: c.name)
@pytest.mark.parametrize("kind", ASSISTANTS)
@pytest.mark.parametrize("K", [1, 3, 15])
def test_rounds_teacher_forced(cfg, kind, K):
    dm, draft = _target(cfg), _assistant(cfg, kind)
    st, ast = dm.stage, draft.stage
    oracle_t, oracle_a = _oracle(cfg), _oracle(_assistant_cfg(cfg, kind), _assistant_seed(kind))
    ids = _prompt(cfg).cuda()
    S, new = ids.shape[1], 32
    st.set_sampling(None)
    st.set_logits_processors(None)
    x = st.prefill(st.embed(ids), 0, 0)
    first = st.ids_dec[0][:1]
    st.head_argmax(x[:, -1, :].contiguous(), first, 0)
    ast.prefill(ast.embed(ids), 0, 0)
    seq = torch.cat([ids, first.view(1, 1)], dim=1).cpu()
    st.prompt_lookup_begin(seq.cuda(), K, 0, S + new, [], assistant=ast)
    per_round, checked = [], 0
    while seq.shape[1] < S + new:
        drafts, emitted = st.verify_round()
        assert len(drafts) == K and 1 <= len(emitted) <= K + 1
        want_d, m_d = oracle_a.generate(seq, K, return_margins=True)
        n = _reliable(m_d)
        assert drafts[:n] == want_d[0, seq.shape[1]:seq.shape[1] + n].tolist(), (seq.shape[1], drafts, want_d)
        want_e, m_e = oracle_t.generate(seq, len(emitted), return_margins=True)
        n_e = _reliable(m_e)
        assert emitted[:n_e] == want_e[0, seq.shape[1]:seq.shape[1] + n_e].tolist(), (seq.shape[1], emitted, want_e)
        # the accepted prefix is the agreeing prefix of the drafts
        a = len(emitted) - 1
        assert emitted[:a] == drafts[:a] and (a == K or len(emitted) == S + new - seq.shape[1]
                                              or emitted[a] != drafts[a])
        checked += n + n_e
        per_round.append(len(emitted))
        seq = torch.cat([seq, torch.tensor([emitted])], dim=1)
    print(f"{cfg.name} {kind} K={K}: tokens per round {per_round}; {checked} draft/emitted tokens oracle-checked")
    assert checked >= 2


# ------------------------------------------------------------------------------------------ generate
class _Streamer:
    def __init__(self):
        self.puts, self.ended = [], False

    def put(self, t):
        self.puts.append(t.clone())

    def end(self):
        self.ended = True


def _teacher_forced(dm, seq, S, margin=MARGIN):
    """argmax of one forward over ``seq`` at the generated positions, and where its top-2 margin exceeds ``margin``"""
    logits = dm(seq[:, :-1]).logits[:, S - 1:].cpu().float()
    top2 = logits.topk(2, -1).values
    return logits.argmax(-1), (top2[..., 0] - top2[..., 1]) > margin


@pytest.mark.parametrize("cfg", CASES, ids=lambda c: c.name)
@pytest.mark.parametrize("kind", ASSISTANTS)
@pytest.mark.parametrize("K", [1, 2, 5, 15])
def test_generate_assisted(cfg, kind, K):
    from tests.test_model_gpu import _check_ids
    dm, draft = _target(cfg), _assistant(cfg, kind)
    ids = _prompt(cfg)
    S, new = ids.shape[1], 40
    ref, margins = _oracle(cfg).generate(ids, new, return_margins=True)
    plain = dm.generate(ids, max_new_tokens=new).cpu()
    stream = _Streamer()
    got = dm.generate(ids, max_new_tokens=new, assistant_model=draft, num_assistant_tokens=K, streamer=stream).cpu()
    steps = dm.timers["assisted_steps"]
    eager = dm.generate(ids, max_new_tokens=new, assistant_model=draft, num_assistant_tokens=K, use_graph=False).cpu()
    assert got.shape == (1, S + new) and torch.equal(got[:, :S], ids)
    assert torch.equal(got, eager)                          # CUDA-graph replay == eager launches, bit for bit
    assert torch.equal(dm.generate(ids, max_new_tokens=new).cpu(), plain)     # plain decoding is left as it was
    n = _check_ids(got, ref, margins, S)
    n_ok = _reliable(margins)
    assert torch.equal(got[:, S:S + n_ok], plain[:, S:S + n_ok])
    tf, safe = _teacher_forced(dm, got, S)
    assert safe.float().mean() > 0.2
    assert torch.equal(tf[safe], got[:, S:][safe])
    assert stream.ended and all(t.numel() == 1 for t in stream.puts)
    assert torch.cat(stream.puts).tolist() == got[0, S:].tolist()
    all_accept = -(-(new - 1) // (K + 1))                   # K+1 tokens a round after the prefill's, the last one cut
    print(f"{cfg.name} {kind} K={K}: {new} tokens in {steps} rounds + the prefill's "
          f"({(new - 1) / max(steps, 1):.2f} tokens per round; all-accept {all_accept}), {n} steps oracle-exact")
    assert all_accept <= steps <= new - 1
    if kind == "same":
        # the assistant IS the model: a draft is rejected only where the two verify paths' last bits split a near tie
        assert steps <= all_accept + int((~safe).sum())
        if bool(safe.all()):
            assert steps == all_accept
    # EOS: the assisted run stops where plain decoding does
    j = next((s for s in range(min(n_ok, new)) if got[0, S + s] not in got[0, S:S + s].tolist() and s >= 3), None)
    if j is not None:
        eos = int(got[0, S + j])
        p = dm.generate(ids, max_new_tokens=new, eos_token_id=eos).cpu()
        g = dm.generate(ids, max_new_tokens=new, eos_token_id=eos, assistant_model=draft, num_assistant_tokens=K).cpu()
        assert torch.equal(g, p) and g.shape[1] == S + j + 1
        assert torch.equal(g, apply_eos(got, S, eos))


def test_mismatched_vocabularies():
    """An assistant with half the model's vocabulary, and a prompt holding ids it cannot embed."""
    cfg = C.TINY_QWEN2
    dm = _target(cfg)
    small = _make(cfg.scaled(vocab=cfg.vocab // 2, n_layers=2))
    ids = synthetic_tokens(cfg, 1, 16)
    ids[0, ::2] = cfg.vocab - 1 - torch.arange(8)           # above the assistant's vocabulary
    plain = dm.generate(ids, max_new_tokens=32).cpu()
    for K in (1, 4, 15):
        got = dm.generate(ids, max_new_tokens=32, assistant_model=small, num_assistant_tokens=K).cpu()
        assert torch.equal(got, plain), K
    # the other way round: drafts the model cannot embed are never accepted
    big = _make(cfg.scaled(vocab=cfg.vocab * 2))
    plain_s = small.generate(ids, max_new_tokens=24).cpu()
    assert torch.equal(small.generate(ids, max_new_tokens=24, assistant_model=big, num_assistant_tokens=3).cpu(), plain_s)


@pytest.mark.parametrize("K", [1, 4])
def test_max_new_boundaries(K):
    cfg = C.TINY_QWEN2
    dm, draft = _target(cfg), _assistant(cfg, "two_layers")
    ids = _prompt(cfg)
    S = ids.shape[1]
    full = dm.generate(ids, max_new_tokens=30, assistant_model=draft, num_assistant_tokens=K).cpu()
    for m in sorted({1, 2, K, K + 1, K + 2, 29}):
        got = dm.generate(ids, max_new_tokens=m, assistant_model=draft, num_assistant_tokens=K).cpu()
        assert got.shape == (1, S + m), m
        assert torch.equal(got, full[:, :S + m]), m
        assert dm.timers["assisted_steps"] <= m - 1


def test_graph_lifetime():
    """Two assistants alternate, with the assistants' own generate in between: every result is its first run's, and
    the model's plain decoding and prompt lookup give what they gave before."""
    cfg = C.TINY_QWEN2_D128
    dm = _make(cfg)
    a, b = _make(cfg), _make(cfg.scaled(n_layers=2))
    ids = _prompt(cfg)
    plain0 = dm.generate(ids, max_new_tokens=24).cpu()
    look0 = dm.generate(ids, max_new_tokens=24, prompt_lookup_num_tokens=3).cpu()
    first = {}
    for it in range(3):
        for name, asst in (("a", a), ("b", b)):
            for K in (2, 5):
                got = dm.generate(ids, max_new_tokens=24, assistant_model=asst, num_assistant_tokens=K).cpu()
                assert torch.equal(got, first.setdefault((name, K), got)), (it, name, K)
            own = asst.generate(ids, max_new_tokens=16).cpu()
            assert torch.equal(own, first.setdefault((name, "own"), own)), (it, name)
    assert sum(k[0] == "assist" for k in dm.stage.graphs) == 2       # the last assistant's graphs only
    assert torch.equal(dm.generate(ids, max_new_tokens=24).cpu(), plain0)
    assert torch.equal(dm.generate(ids, max_new_tokens=24, prompt_lookup_num_tokens=3).cpu(), look0)
    # the assistant's default K, and an attention mask with leading zeros
    got = dm.generate(ids, max_new_tokens=24, assistant_model=a).cpu()
    padded = torch.cat([torch.zeros(1, 3, dtype=torch.int64), ids], dim=1)
    mask = torch.cat([torch.zeros(1, 3, dtype=torch.int64), torch.ones_like(ids)], dim=1)
    got_p = dm.generate(padded, attention_mask=mask, max_new_tokens=24, assistant_model=a).cpu()
    assert torch.equal(got_p[:, 3:], got) and torch.equal(got_p[:, :3], padded[:, :3])


def test_full_size_qwen25_7b_with_05b_assistant():
    """Qwen2.5-7B with a Qwen2.5-0.5B assistant at full size (device-initialised weights): head dims 128 / 64 and
    vocabularies 152,064 / 151,936 differ.  Against plain decoding and one forward over the final sequence, graph
    against eager."""
    dm = _make(C.QWEN25_7B, init="device")
    draft = _make(C.QWEN25_05B, init="device")
    ids = synthetic_tokens(C.QWEN25_7B, 1, 32)
    S, new = ids.shape[1], 48
    plain = dm.generate(ids, max_new_tokens=new).cpu()
    for K in (2, 5):
        got = dm.generate(ids, max_new_tokens=new, assistant_model=draft, num_assistant_tokens=K).cpu()
        steps = dm.timers["assisted_steps"]
        eager = dm.generate(ids, max_new_tokens=new, assistant_model=draft, num_assistant_tokens=K, use_graph=False).cpu()
        assert torch.equal(got, eager) and got.shape == plain.shape
        for name, seq in (("plain", plain), (f"K={K}", got)):
            # the logits are bf16: at the 7B model's logit magnitudes one bf16 step is ~0.03-0.06, and the decode,
            # verify and prefill paths round differently through 28 layers, so a resolvable margin is several steps
            tf, safe = _teacher_forced(dm, seq, S, MARGIN_FULL)
            wrong = (tf != seq[:, S:])[0].nonzero().flatten().tolist()
            print(f"{name}: {safe.float().mean():.2f} of the positions resolvable, teacher-forced argmax differs at {wrong}")
            assert safe.float().mean() > 0.2
            assert torch.equal(tf[safe], seq[:, S:][safe])
        diff = (got != plain)[0, S:].nonzero()
        print(f"Qwen2.5-7B + 0.5B K={K}: {new} tokens in {steps} rounds ({(new - 1) / max(steps, 1):.2f} tokens per "
              f"round); first divergence from plain decoding: {int(diff[0]) if diff.numel() else None}")
