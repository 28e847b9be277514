"""Host side of left-padded generation: mask -> (trimmed width, per-row key starts), and the grouped path that stages
without per-row key starts (``supports_kv_start``) still take."""
import pytest
import torch

from tensorlink_b200.ml import module as M


def test_left_pad_starts_from_mask():
    assert M._left_pad_starts(torch.ones(2, 5, dtype=torch.int64)) is None            # nothing padded: the plain path
    mask = torch.tensor([[0, 0, 1, 1, 1], [1, 1, 1, 1, 1], [0, 0, 0, 0, 1]])
    assert M._left_pad_starts(mask) == (0, [2, 0, 4])
    # two columns are pad in every row: they are dropped, the starts count what is left
    mask = torch.tensor([[0, 0, 0, 1, 1], [0, 0, 1, 1, 1], [0, 0, 0, 0, 1]])
    assert M._left_pad_starts(mask) == (2, [1, 0, 2])
    assert M._left_pad_starts(mask.bool()) == (2, [1, 0, 2])
    for bad in (torch.tensor([[1, 1, 0], [1, 1, 1]]), torch.tensor([[0, 1, 0], [1, 1, 1]]), torch.tensor([[0, 0], [1, 1]])):
        with pytest.raises(NotImplementedError):
            M._left_pad_starts(bad)


class _Link:
    rank, world, first, last = 0, 1, True, True

    def broadcast_object(self, o, *a):
        return o


class _Stage:
    """A stage without per-row key starts (as the CPU oracle stage of the pipeline tests)."""
    max_batch, max_seq = 4, 64


def test_stage_without_kv_start_takes_the_grouped_path():
    dm = M.DistributedModel.__new__(M.DistributedModel)
    torch.nn.Module.__init__(dm)
    dm.link, dm.stage, dm.cfg, dm.world = _Link(), _Stage(), None, 1
    seen = {}

    def grouped(input_ids, req):
        seen.update(groups=req.groups, shape=req.shape)
        return "grouped"

    dm._generate_left_padded = grouped
    dm._generate_batch = lambda *a, **k: pytest.fail("the one-run path needs supports_kv_start")
    ids = torch.arange(8).view(2, 4)
    mask = torch.tensor([[0, 1, 1, 1], [1, 1, 1, 1]])
    assert dm.generate(ids, attention_mask=mask, max_new_tokens=2) == "grouped"
    assert seen == {"groups": {3: [0], 4: [1]}, "shape": (2, 4)}

    _Stage.supports_kv_start = True
    try:
        got = {}
        dm._generate_left_padded = lambda *a, **k: pytest.fail("a stage with supports_kv_start runs the batch once")
        dm._generate_batch = lambda input_ids, req: (got.update(ids=input_ids, kv_start=req.kv_start), input_ids)[1]
        mask = torch.tensor([[0, 0, 1, 1], [0, 1, 1, 1]])
        out = dm.generate(ids, attention_mask=mask, max_new_tokens=2)
        assert got["kv_start"] == [1, 0] and torch.equal(got["ids"], ids[:, 1:])
        assert torch.equal(out, ids)                     # the dropped pad column returns in the result
    finally:
        del _Stage.supports_kv_start
