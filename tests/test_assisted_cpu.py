"""``generate(assistant_model=draft, num_assistant_tokens=K)``: keyword validation on the host, before any stage work.

The CPU oracle stage stands in for the CUDA one on the model and on its assistant (tests/oracle_stage.py, through the
``_stage_factory`` hook): every error below must be raised before either stage embeds or prefills anything."""
import pytest
import torch

from tensorlink_b200.ml import DistributedModel
from tensorlink_b200.ml import configs as C
from tensorlink_b200.ml import module as M
from tensorlink_b200.p2p.link import StageLink
from tests.oracle_stage import OracleStage

CFG = C.TINY_QWEN2
MAX_SEQ = 64


class _Spy(OracleStage):
    """Counts the stage work a generate call does, on every model."""
    calls = 0

    def embed(self, ids):
        _Spy.calls += 1
        return super().embed(ids)

    def prefill(self, hidden, past_len=0, slot=0):
        _Spy.calls += 1
        return super().prefill(hidden, past_len, slot)


def _model(cfg=CFG, max_seq=MAX_SEQ):
    return DistributedModel(cfg, training=False, max_batch=2, max_seq=max_seq, _stage_factory=_Spy, device="cpu",
                            link=StageLink(0, 1))


@pytest.fixture(scope="module")
def dm():
    return _model()


@pytest.fixture(scope="module")
def draft():
    return _model(CFG.scaled(n_layers=2))


def _ids(rows=1, S=8):
    return torch.arange(rows * S, dtype=torch.int64).view(rows, S) % CFG.vocab


def _raises(dm, exc, match, ids=None, **kw):
    _Spy.calls = 0
    with pytest.raises(exc, match=match):
        dm.generate(_ids() if ids is None else ids, **kw)
    assert _Spy.calls == 0, "stage work before the keyword check"


def test_prompt_lookup_and_assistant_together(dm, draft):
    # checked before anything looks at the assistant: even a bad one names the combination
    for a in (draft, object()):
        _raises(dm, NotImplementedError, "assistant_model together with prompt_lookup_num_tokens", assistant_model=a,
                prompt_lookup_num_tokens=3, num_assistant_tokens=0, max_new_tokens=4)


@pytest.mark.parametrize("a", [object(), torch.nn.Linear(2, 2), "Qwen/Qwen2.5-0.5B"])
def test_assistant_must_be_a_distributed_model(dm, a):
    _raises(dm, TypeError, r"DistributedModel\(hf_model, training=False\)", assistant_model=a, num_assistant_tokens=0,
            max_new_tokens=4)


def test_model_is_not_its_own_assistant(dm):
    _raises(dm, ValueError, "the model itself", assistant_model=dm, max_new_tokens=4)


@pytest.mark.parametrize("K", [0, -1, 16, 20, 2.0, "3", True])
def test_num_assistant_tokens_in_range(dm, draft, K):
    _raises(dm, ValueError, "num_assistant_tokens has to be an integer in 1..15", assistant_model=draft,
            num_assistant_tokens=K, max_new_tokens=4, do_sample=True)          # ValueError before NotImplementedError


def test_one_row_only(dm, draft):
    _raises(dm, ValueError, "one row at a time", ids=_ids(rows=2), assistant_model=draft, max_new_tokens=4)


def test_cache_of_either_model_must_hold_the_last_verify_step():
    target, small = _model(), _model(CFG.scaled(n_layers=2), max_seq=32)
    # 8 + 41 + 15 = 64 fits the model, not the assistant
    _raises(target, ValueError, "max_seq of the assistant", assistant_model=small, num_assistant_tokens=15,
            max_new_tokens=41)
    _raises(target, ValueError, "max_seq of the model", assistant_model=_model(CFG.scaled(n_layers=2)),
            num_assistant_tokens=15, max_new_tokens=42)
    _raises(small, ValueError, "max_seq of the model", assistant_model=target, num_assistant_tokens=2, max_new_tokens=23)


@pytest.mark.parametrize("kw,match", [
    (dict(do_sample=True), "do_sample"),
    (dict(repetition_penalty=1.2), "repetition_penalty"),
    (dict(no_repeat_ngram_size=3), "repetition_penalty"),
    (dict(min_new_tokens=2, eos_token_id=5), "repetition_penalty"),
    (dict(), "CUDA stage"),                                  # the oracle stage is not the CUDA one
])
def test_unsupported_combinations(dm, draft, kw, match):
    _raises(dm, NotImplementedError, match, assistant_model=draft, num_assistant_tokens=3, max_new_tokens=4, **kw)


def test_more_than_eight_eos_ids_need_no_device_slot(dm, draft):
    # the assisted step has no EOS ids on the device: the first complaint is the stage, not the count
    _raises(dm, NotImplementedError, "CUDA stage", assistant_model=draft, max_new_tokens=4, eos_token_id=list(range(9)))


def test_pipelines_and_devices(dm, draft, monkeypatch):
    from tensorlink_b200.ml import stage as S
    monkeypatch.setattr(draft, "world", 2)
    _raises(dm, NotImplementedError, "more than one stage", assistant_model=draft, max_new_tokens=4)
    monkeypatch.setattr(draft, "world", 1)
    monkeypatch.setattr(dm, "world", 2)
    _raises(dm, NotImplementedError, "more than one stage", assistant_model=draft, max_new_tokens=4)
    monkeypatch.setattr(dm, "world", 1)
    # past the CUDA-stage check (the spy stands in for it), an assistant on another device
    monkeypatch.setattr(S, "CudaStage", _Spy)
    monkeypatch.setattr(draft.stage, "device", torch.device("cpu", 1))
    _raises(dm, NotImplementedError, "assistant_model on cpu:1", assistant_model=draft, max_new_tokens=4)
    monkeypatch.setattr(draft.stage, "device", torch.device("cpu"))
    got = M._assisted(dm, draft, None, (1, 8), 4)
    assert got == {"K": M.ASSISTED_DEFAULT_K, "ngram": 0, "assistant": draft.stage}
    assert M._assisted(dm, draft, 15, (1, 8), 41)["K"] == 15


@pytest.mark.parametrize("kw", [dict(num_assistant_tokens_schedule="heuristic"),
                                dict(num_assistant_tokens_schedule="heuristic_transient"),
                                dict(assistant_confidence_threshold=0.4)])
def test_schedules_and_confidence_stay_unsupported(dm, draft, kw):
    _raises(dm, NotImplementedError, next(iter(kw)), assistant_model=draft, max_new_tokens=4, **kw)


def test_num_assistant_tokens_alone_stays_unsupported(dm):
    _raises(dm, NotImplementedError, "num_assistant_tokens", num_assistant_tokens=3, max_new_tokens=4)


def test_neutral_values_are_the_same_as_leaving_them_out(dm):
    ids = _ids()
    a = dm.generate(ids, max_new_tokens=5)
    for kw in (dict(assistant_model=None), dict(num_assistant_tokens_schedule="constant"),
               dict(num_assistant_tokens_schedule=None), dict(assistant_confidence_threshold=None),
               dict(assistant_model=None, num_assistant_tokens_schedule="constant", assistant_confidence_threshold=None)):
        assert torch.equal(dm.generate(ids, max_new_tokens=5, **kw), a), kw
