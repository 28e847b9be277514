"""``generate(do_sample=True)`` with ``assistant_model`` or ``prompt_lookup_num_tokens``: validation on the host.

The CPU oracle stage stands in for the CUDA one (tests/oracle_stage.py): past the CUDA-stage check (monkeypatched),
sampled drafts pass validation; bad sampling values still raise ValueError and logits processors with drafts still
raise NotImplementedError, all before any stage work."""
import pytest
import torch

from tensorlink_b200.ml import DistributedModel
from tensorlink_b200.ml import configs as C
from tensorlink_b200.ml import module as M
from tensorlink_b200.p2p.link import StageLink
from tests.oracle_stage import OracleStage

CFG = C.TINY_QWEN2
SAMPLING = {"temperature": 0.8, "top_k": 20, "top_p": 0.9, "seed": 3}


class _Spy(OracleStage):
    calls = 0

    def embed(self, ids):
        _Spy.calls += 1
        return super().embed(ids)

    def prefill(self, hidden, past_len=0, slot=0):
        _Spy.calls += 1
        return super().prefill(hidden, past_len, slot)


def _model(cfg=CFG):
    return DistributedModel(cfg, training=False, max_batch=2, max_seq=64, _stage_factory=_Spy, device="cpu",
                            link=StageLink(0, 1))


@pytest.fixture(scope="module")
def dm():
    return _model()


@pytest.fixture(scope="module")
def draft():
    return _model(CFG.scaled(n_layers=2))


def _raises(dm, exc, match, **kw):
    _Spy.calls = 0
    with pytest.raises(exc, match=match):
        dm.generate(torch.arange(8, dtype=torch.int64).view(1, 8), max_new_tokens=4, **kw)
    assert _Spy.calls == 0, "stage work before the keyword check"


def test_sampled_drafts_pass_validation(dm, draft, monkeypatch):
    from tensorlink_b200.ml import stage as S
    monkeypatch.setattr(S, "CudaStage", _Spy)
    assert M._assisted(dm, draft, 3, (1, 8), 4, sampling=SAMPLING) == {"K": 3, "ngram": 0, "assistant": draft.stage}
    assert M._assisted(dm, draft, None, (1, 8), 4, sampling=SAMPLING)["K"] == M.ASSISTED_DEFAULT_K
    assert M._prompt_lookup(3, None, (1, 8), 4, 64, sampling=SAMPLING, stage=dm.stage) == {"K": 3, "ngram": 2}


@pytest.mark.parametrize("source", [dict(prompt_lookup_num_tokens=3), "assistant"])
def test_sampled_drafts_need_the_cuda_stage(dm, draft, source):
    kw = dict(assistant_model=draft, num_assistant_tokens=3) if source == "assistant" else source
    _raises(dm, NotImplementedError, "do_sample=True needs the CUDA stage", do_sample=True, **kw)


@pytest.mark.parametrize("bad", [dict(temperature=0.0), dict(temperature=-1.0), dict(top_p=0.0), dict(top_p=1.5),
                                 dict(top_k=-1)])
@pytest.mark.parametrize("source", [dict(prompt_lookup_num_tokens=3), "assistant"])
def test_invalid_sampling_values_raise_value_error(dm, draft, bad, source):
    kw = dict(assistant_model=draft, num_assistant_tokens=3) if source == "assistant" else source
    _raises(dm, ValueError, "invalid sampling parameters", do_sample=True, **bad, **kw)


@pytest.mark.parametrize("procs", [dict(repetition_penalty=1.2), dict(no_repeat_ngram_size=2),
                                   dict(min_new_tokens=2, eos_token_id=5)])
@pytest.mark.parametrize("source", [dict(prompt_lookup_num_tokens=3), "assistant"])
def test_logits_processors_with_sampled_drafts_still_raise(dm, draft, procs, source, monkeypatch):
    from tensorlink_b200.ml import stage as S
    monkeypatch.setattr(S, "CudaStage", _Spy)                # the stage is not what is missing
    kw = dict(assistant_model=draft, num_assistant_tokens=3) if source == "assistant" else source
    _raises(dm, NotImplementedError, "repetition_penalty", do_sample=True, **procs, **kw)


def test_several_rows_and_stages_still_raise(dm, draft, monkeypatch):
    _Spy.calls = 0
    with pytest.raises(ValueError, match="one row at a time"):
        dm.generate(torch.zeros(2, 8, dtype=torch.int64), max_new_tokens=4, do_sample=True, assistant_model=draft)
    monkeypatch.setattr(draft, "world", 2)
    _raises(dm, NotImplementedError, "more than one stage", do_sample=True, assistant_model=draft)
    with pytest.raises(NotImplementedError, match="more than one stage"):
        M._prompt_lookup(3, None, (1, 8), 4, 64, sampling=SAMPLING, world=2)
