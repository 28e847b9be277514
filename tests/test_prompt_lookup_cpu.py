"""``generate(prompt_lookup_num_tokens=K)``: keyword validation on the host, before any stage work.

The CPU oracle stage stands in for the CUDA one (tests/oracle_stage.py, through the ``_stage_factory`` hook): every
ValueError / NotImplementedError below must be raised before the stage embeds or prefills anything."""
import pytest
import torch

from tensorlink_b200.ml import DistributedModel
from tensorlink_b200.ml import configs as C
from tensorlink_b200.ml.module import _prompt_lookup
from tensorlink_b200.p2p.link import StageLink
from tests.oracle_stage import OracleStage

CFG = C.TINY_QWEN2
MAX_SEQ = 64


class _Spy(OracleStage):
    """Counts the stage work a generate call does."""
    calls = 0

    def embed(self, ids):
        _Spy.calls += 1
        return super().embed(ids)

    def prefill(self, hidden, past_len=0, slot=0):
        _Spy.calls += 1
        return super().prefill(hidden, past_len, slot)


@pytest.fixture(scope="module")
def dm():
    return DistributedModel(CFG, training=False, max_batch=2, max_seq=MAX_SEQ, _stage_factory=_Spy, device="cpu",
                            link=StageLink(0, 1))


def _ids(rows=1, S=8):
    return torch.arange(rows * S, dtype=torch.int64).view(rows, S) % CFG.vocab


def _raises(dm, exc, match, ids=None, **kw):
    _Spy.calls = 0
    with pytest.raises(exc, match=match):
        dm.generate(_ids() if ids is None else ids, **kw)
    assert _Spy.calls == 0, "stage work before the keyword check"


@pytest.mark.parametrize("K", [0, -1, 2.0, "3", True])
def test_num_tokens_must_be_a_positive_integer(dm, K):
    _raises(dm, ValueError, "prompt_lookup_num_tokens has to be a positive integer", prompt_lookup_num_tokens=K,
            max_new_tokens=4)


@pytest.mark.parametrize("n", [0, -2, 1.5, False])
def test_ngram_size_must_be_a_positive_integer(dm, n):
    _raises(dm, ValueError, "max_matching_ngram_size has to be a positive integer", prompt_lookup_num_tokens=3,
            max_matching_ngram_size=n, max_new_tokens=4)


def test_at_most_15_drafts(dm):
    _raises(dm, ValueError, "at most 15 drafts", prompt_lookup_num_tokens=16, max_new_tokens=4)


def test_one_row_only(dm):
    _raises(dm, ValueError, "one row at a time", ids=_ids(rows=2), prompt_lookup_num_tokens=3, max_new_tokens=4)


def test_cache_must_hold_the_last_verify_step(dm):
    # S + max_new + K > max_seq: the last step writes K+1 slots from position S + max_new - 2
    _raises(dm, ValueError, "max_seq", prompt_lookup_num_tokens=10, max_new_tokens=MAX_SEQ - 8 - 9)


@pytest.mark.parametrize("kw,match", [
    (dict(do_sample=True), "do_sample"),
    (dict(repetition_penalty=1.2), "repetition_penalty"),
    (dict(no_repeat_ngram_size=3), "repetition_penalty"),
    (dict(min_new_tokens=2, eos_token_id=5), "repetition_penalty"),
    (dict(eos_token_id=list(range(9))), "more than 8 EOS ids"),
    (dict(), "CUDA stage"),                                  # the oracle stage is not the CUDA one
])
def test_unsupported_combinations(dm, kw, match):
    _raises(dm, NotImplementedError, match, prompt_lookup_num_tokens=3, max_new_tokens=4, **kw)


def test_assistant_model_stays_unsupported(dm):
    _raises(dm, NotImplementedError, "assistant_model", prompt_lookup_num_tokens=3, assistant_model=object(),
            max_new_tokens=4)


def test_ngram_size_alone_stays_unsupported(dm):
    _raises(dm, NotImplementedError, "max_matching_ngram_size", max_matching_ngram_size=3, max_new_tokens=4)


def test_none_is_the_same_as_leaving_it_out(dm):
    ids = _ids()
    a = dm.generate(ids, max_new_tokens=5)
    b = dm.generate(ids, max_new_tokens=5, prompt_lookup_num_tokens=None)
    assert torch.equal(a, b)


def test_validation_helper():
    shape = (1, 8)
    assert _prompt_lookup(None, None, shape, 4, 64) is None
    with pytest.raises(NotImplementedError, match="more than one stage"):
        _prompt_lookup(3, None, shape, 4, 64, world=2)
    # every ValueError comes before what is not implemented
    with pytest.raises(ValueError, match="one row"):
        _prompt_lookup(3, 2, (2, 8), 4, 64, sampling={"temperature": 1.0}, world=2)
    with pytest.raises(ValueError, match="max_seq"):
        _prompt_lookup(15, 2, shape, 42, 64)
    with pytest.raises(NotImplementedError, match="CUDA stage"):
        _prompt_lookup(15, 2, shape, 41, 64)                       # 8 + 41 + 15 = 64 fits
