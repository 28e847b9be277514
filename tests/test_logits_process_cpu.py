"""Host side of the logits processors in ``DistributedModel.generate``: keyword validation, the refusal paths, and the
starting history that keeps the pad columns a left-padded run drops."""
import pytest
import torch

from tensorlink_b200.ml import module as M


class _Link:
    rank, world, first, last = 0, 1, True, True

    def broadcast_object(self, o, *a):
        return o


class _Stage:
    """A stage without the logits processors (as the CPU oracle stage of the pipeline tests)."""
    max_batch, max_seq = 4, 64


def _dm(stage):
    dm = M.DistributedModel.__new__(M.DistributedModel)
    torch.nn.Module.__init__(dm)
    dm.link, dm.stage, dm.cfg, dm.world = _Link(), stage, None, 1
    return dm


def test_keyword_validation():
    assert M._logits_processors() is None
    assert M._logits_processors(1.0, 0, 0) is None and M._logits_processors(1, None, None) is None
    assert M._logits_processors(1.2) == {"penalty": 1.2, "ngram": 0, "min_new": 0, "eos": []}
    assert M._logits_processors(0.5, 3, 2) == {"penalty": 0.5, "ngram": 3, "min_new": 2, "eos": []}
    assert M._logits_processors(1.0, 0, 2, torch.tensor([7, 9]))["eos"] == [7, 9]
    assert M._logits_processors(1.2, 0, 0, 7)["eos"] == []             # no min_new_tokens: no EOS id is held back
    for bad in (dict(repetition_penalty=0.0), dict(repetition_penalty=-1.0), dict(repetition_penalty="1.2"),
                dict(no_repeat_ngram_size=-1), dict(no_repeat_ngram_size=1.5), dict(no_repeat_ngram_size=True),
                dict(min_new_tokens=-2), dict(min_new_tokens=2.0)):
        with pytest.raises(ValueError):
            M._logits_processors(**bad)


def test_forward_and_unconsumed_keywords_still_refuse():
    with pytest.raises(NotImplementedError):
        M._check_unconsumed({"repetition_penalty": 1.2}, "DistributedModel.forward")
    with pytest.raises(NotImplementedError):
        M._check_unconsumed({"no_repeat_ngram_size": 2}, "DistributedModel.forward")
    for kw in ({"presence_penalty": 0.5}, {"bad_words_ids": [[1]]}, {"min_length": 3}):
        with pytest.raises(NotImplementedError):
            M._check_unconsumed(kw, "DistributedModel.generate")


def test_too_many_eos_ids_raise_before_any_work():
    """Checked on every rank from its own keywords, before the first collective (the head stage alone must not raise
    while the other ranks go on into the prefill)."""
    dm = _dm(_ProcStage())
    dm._generate_batch = lambda *a, **k: pytest.fail("the run started")
    with pytest.raises(NotImplementedError, match="EOS ids"):
        dm.generate(torch.arange(8).view(2, 4), max_new_tokens=2, min_new_tokens=3, eos_token_id=list(range(9)))
    assert M._logits_processors(1.0, 0, 3, list(range(8)))["eos"] == list(range(8))


def test_invalid_values_raise_before_any_work():
    dm = _dm(_Stage())
    dm._generate_batch = lambda *a, **k: pytest.fail("invalid keywords reached the run")
    ids = torch.arange(8).view(2, 4)
    with pytest.raises(ValueError):
        dm.generate(ids, max_new_tokens=2, repetition_penalty=0)
    with pytest.raises(ValueError):
        dm.generate(ids, max_new_tokens=2, no_repeat_ngram_size=-3)


def test_stage_without_support_raises():
    dm = _dm(_Stage())
    dm._generate_batch = lambda *a, **k: pytest.fail("the stage cannot apply the processors")
    dm._generate_left_padded = lambda *a, **k: pytest.fail("the stage cannot apply the processors")
    ids = torch.arange(8).view(2, 4)
    for kw in (dict(repetition_penalty=1.2), dict(no_repeat_ngram_size=2), dict(min_new_tokens=3, eos_token_id=1)):
        with pytest.raises(NotImplementedError, match="CUDA stage"):
            dm.generate(ids, max_new_tokens=2, **kw)
        with pytest.raises(NotImplementedError, match="CUDA stage"):      # the grouped left-padded path too
            dm.generate(ids, attention_mask=torch.tensor([[0, 1, 1, 1], [1, 1, 1, 1]]), max_new_tokens=2, **kw)


def test_grouped_left_padded_path_refuses_the_processors():
    """A stage with the processors but without per-row key starts would run one group per real length, each without
    the pad columns of its history: refused instead of silently computing something else."""
    class _NoKvStart(_Stage):
        def set_logits_processors(self, procs, length=0):
            pass

    dm = _dm(_NoKvStart())
    dm._generate_left_padded = lambda *a, **k: pytest.fail("the grouped runs would drop the processors' pads")
    with pytest.raises(NotImplementedError, match="supports_kv_start"):
        dm.generate(torch.arange(8).view(2, 4), attention_mask=torch.tensor([[0, 1, 1, 1], [1, 1, 1, 1]]),
                    max_new_tokens=2, repetition_penalty=1.2)


class _ProcStage(_Stage):
    supports_kv_start = True

    def set_logits_processors(self, procs, length=0):
        pass


def test_history_keeps_the_dropped_pad_columns():
    dm = _dm(_ProcStage())
    seen = {}

    def run(input_ids, req):
        seen.update(ids=input_ids, kv_start=req.kv_start, procs=req.procs, history=req.history)
        return input_ids

    dm._generate_batch = run
    ids = torch.tensor([[9, 9, 4, 5], [9, 6, 7, 8]])
    mask = torch.tensor([[0, 0, 1, 1], [0, 1, 1, 1]])
    dm.generate(ids, attention_mask=mask, max_new_tokens=2, repetition_penalty=1.3)
    assert torch.equal(seen["ids"], ids[:, 1:]) and seen["kv_start"] == [1, 0]
    prompt = seen["history"]
    assert seen["procs"] == {"penalty": 1.3, "ngram": 0, "min_new": 0, "eos": []}
    assert torch.equal(prompt, ids)                           # HF counts every column, the pad in every row included
    dm.generate(ids, max_new_tokens=2)
    assert seen["procs"] is None                              # neutral values: the processors stay off
