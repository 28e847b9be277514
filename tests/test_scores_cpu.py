"""``generate(return_dict_in_generate=True, output_scores=..., output_logits=...)`` on the host: keyword handling and the
refusals (checked before any stage work), ``compute_transition_scores`` against HF's own function, and the CPU
reference of the scores (tests/scores_ref.py) the GPU tests compare with."""
import types

import pytest
import torch

from tensorlink_b200.ml import DistributedModel
from tensorlink_b200.ml import configs as C
from tensorlink_b200.ml import module as M
from tensorlink_b200.p2p.link import StageLink
from tests.oracle_stage import OracleStage
from tests.scores_ref import hf_processed, hf_warped_scores, kept_scores

CFG = C.TINY_QWEN2


class _Spy(OracleStage):
    calls = 0

    def embed(self, ids):
        _Spy.calls += 1
        return super().embed(ids)


class _GroupedSpy(_Spy):
    """A stage that could log scores but has no per-row key starts: left-padded batches run as grouped calls."""
    supports_kv_start = False

    def set_score_log(self, *a, **k):
        raise AssertionError("not reached")


def _model(factory=_Spy):
    return DistributedModel(CFG, training=False, max_batch=4, max_seq=64, _stage_factory=factory, device="cpu",
                            link=StageLink(0, 1))


@pytest.fixture(scope="module")
def dm():
    return _model()


def _ids(rows=1, S=6):
    return torch.arange(rows * S, dtype=torch.int64).view(rows, S) % CFG.vocab


def test_output_flags():
    assert M._output_flags() is None
    for v in (None, False):                          # without return_dict_in_generate=True the output flags are ignored
        assert M._output_flags(v, True, True) is None
        assert M._output_flags(v, None, False) is None
    assert M._output_flags(True) == {"scores": False, "logits": False}
    assert M._output_flags(True, True, None) == {"scores": True, "logits": False}
    assert M._output_flags(True, False, True) == {"scores": False, "logits": True}
    for bad in ({"return_dict_in_generate": 1}, {"output_scores": "yes"}, {"output_logits": 0}):
        with pytest.raises(ValueError):
            M._output_flags(**bad)


def test_flags_without_return_dict_return_the_tensor(dm):
    plain = dm.generate(_ids(), max_new_tokens=3)
    for kw in (dict(output_scores=True), dict(output_logits=True, return_dict_in_generate=False),
               dict(output_scores=None, output_logits=False, return_dict_in_generate=None)):
        got = dm.generate(_ids(), max_new_tokens=3, **kw)
        assert isinstance(got, torch.Tensor) and torch.equal(got, plain)
    # the other output flags stay neutral-only
    for kw in (dict(output_attentions=True), dict(output_hidden_states=True)):
        with pytest.raises(NotImplementedError):
            dm.generate(_ids(), max_new_tokens=2, return_dict_in_generate=True, **kw)


def _raises(dm, match, ids=None, **kw):
    _Spy.calls = 0
    with pytest.raises(NotImplementedError, match=match):
        dm.generate(_ids() if ids is None else ids, max_new_tokens=2, return_dict_in_generate=True, output_scores=True, **kw)
    assert _Spy.calls == 0, "stage work before the keyword check"


def test_refusals(dm):
    _raises(dm, "prompt_lookup_num_tokens / assistant_model", prompt_lookup_num_tokens=2)
    _raises(dm, "prompt_lookup_num_tokens / assistant_model", assistant_model=_model())
    _raises(dm, "needs the CUDA stage")
    _raises(dm, "needs the CUDA stage", do_sample=True)
    grouped = _model(_GroupedSpy)
    ids = _ids(2, 5)
    mask = torch.tensor([[0, 0, 1, 1, 1], [1, 1, 1, 1, 1]])
    _raises(grouped, "left-padded batch", ids=ids, attention_mask=mask)


def _hf_transition(sequences, scores, normalize, V):
    from transformers.generation.utils import GenerationMixin
    text = types.SimpleNamespace(vocab_size=V)
    fake = types.SimpleNamespace(config=types.SimpleNamespace(get_text_config=lambda: text))
    return GenerationMixin.compute_transition_scores(fake, sequences, scores, normalize_logits=normalize)


@pytest.mark.parametrize("B,T,V", [(1, 1, 7), (3, 5, 50), (2, 9, 1000)])
def test_transition_scores_equal_hf(dm, B, T, V):
    g = torch.Generator().manual_seed(B * 100 + T)
    S = 4
    seq = torch.randint(0, V, (B, S + T), generator=g)
    scores = []
    for c in range(T):
        s = torch.randn(B, V, generator=g) * 3
        s[torch.rand(B, V, generator=g) < 0.3] = float("-inf")         # warped rows
        s[torch.arange(B), seq[:, S + c]] = torch.randn(B, generator=g)  # the emitted token stays finite
        scores.append(s)
    for normalize in (False, True):
        got = dm.compute_transition_scores(seq, tuple(scores), normalize_logits=normalize)
        want = _hf_transition(seq, tuple(scores), normalize, V)
        assert got.shape == (B, T)
        assert torch.equal(got, want), normalize
    assert torch.equal(dm.compute_transition_scores(seq, tuple(scores)),
                       torch.stack([scores[c][torch.arange(B), seq[:, S + c]] for c in range(T)], 1))


def test_reference_processors_and_warpers():
    g = torch.Generator().manual_seed(5)
    V = 200
    logits = (torch.randn(2, V, generator=g) * 3).bfloat16()
    hist = [torch.tensor([3, 9, 3, 17, 9, 3]), torch.tensor([1, 2, 1])]
    assert torch.equal(hf_processed(logits, hist), logits.float())          # neutral processors: the fp32 logits
    p = hf_processed(logits, hist, penalty=1.5, ngram=2)
    x = logits.float()
    assert p[0, 3] == (x[0, 3] / 1.5 if x[0, 3] > 0 else x[0, 3] * 1.5)   # seen: penalised
    assert p[0, 3] != x[0, 3] and p[0, 4] == x[0, 4]
    for r, t in ((0, 9), (0, 17), (1, 2)):                                   # "3 9", "3 17" and "1 2" would repeat
        assert p[r, t] == float("-inf")
    w = hf_warped_scores(p, 0.7, 20, 0.9)
    kept = torch.isfinite(w)
    assert 1 <= int(kept[0].sum()) <= 20
    assert torch.equal(w, kept_scores(p, kept, 0.7))                        # HF's warped row: x / T where kept
    assert torch.equal(hf_warped_scores(p), p)
