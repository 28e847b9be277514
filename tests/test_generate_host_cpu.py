"""Host-side pieces of ``DistributedModel.generate`` that need no device: HF keyword screening, attention-mask
classification (left padding), EOS bookkeeping — and the timeline model used to choose the training schedule."""
import importlib.util
import os

import pytest
import torch

from tensorlink_b200.ml import module as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_left_pad_groups_classifies_masks():
    full = torch.ones(3, 5, dtype=torch.int64)
    assert M._left_pad_groups(full) is None                                   # nothing padded: the plain path
    mask = torch.tensor([[0, 0, 1, 1, 1], [1, 1, 1, 1, 1], [0, 0, 1, 1, 1], [0, 0, 0, 0, 1]])
    assert M._left_pad_groups(mask) == {3: [0, 2], 5: [1], 1: [3]}            # rows of equal real length run together
    assert M._left_pad_groups(mask.bool()) == {3: [0, 2], 5: [1], 1: [3]}
    for bad in (torch.tensor([[1, 1, 0, 0]]),                                  # right padding
                torch.tensor([[0, 1, 0, 1]]),                                  # a hole
                torch.tensor([[0, 0, 0, 0], [1, 1, 1, 1]])):                   # an empty row
        with pytest.raises(NotImplementedError):
            M._left_pad_groups(bad)


def test_unconsumed_hf_keywords_raise_unless_neutral():
    M._check_unconsumed({}, "generate")
    M._check_unconsumed({"use_cache": True, "num_beams": 1, "return_dict_in_generate": False}, "generate")   # neutral values pass
    for kw in ({"num_beams": 4}, {"repetition_penalty": 1.2}, {"no_such_keyword": 1}):
        with pytest.raises((NotImplementedError, TypeError)):
            M._check_unconsumed(dict(kw), "generate")


def test_eos_bookkeeping():
    assert M._eos_list(None) == [] and M._eos_list(7) == [7] and M._eos_list([7, 9]) == [7, 9]
    assert M._eos_list(torch.tensor([3, 4])) == [3, 4]
    toks = torch.tensor([[1, 7, 2, 2], [5, 5, 9, 1]])
    assert M._all_rows_finished(toks, [7, 9]) and not M._all_rows_finished(toks, [7]) and not M._all_rows_finished(toks[:, :1], [7, 9])
    # apply_eos: everything after a row's first EOS becomes pad, the result ends where the LAST row finished
    res = torch.tensor([[11, 12, 1, 7, 2, 2], [13, 14, 5, 5, 9, 1]])
    out = M.apply_eos(res, 2, eos_token_id=[7, 9], pad_token_id=0)
    assert out.tolist() == [[11, 12, 1, 7, 0], [13, 14, 5, 5, 9]]
    assert torch.equal(M.apply_eos(res, 2), res)                               # no EOS id: untouched
    assert M.apply_eos(res, 2, eos_token_id=99).shape == res.shape            # never emitted: full length


def test_attention_mask_check_for_forward():
    M._check_attention_mask(None, (2, 4))
    M._check_attention_mask(torch.ones(2, 4), (2, 4))
    with pytest.raises(NotImplementedError):
        M._check_attention_mask(torch.tensor([[0, 1, 1, 1], [1, 1, 1, 1]]), (2, 4))


def _pipeline_model():
    spec = importlib.util.spec_from_file_location("pipeline_model", os.path.join(ROOT, "tools", "pipeline_model.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_timeline_model_reproduces_the_measured_schedules():
    """tools/pipeline_model.py against fixed schedule step times (a regression fixture for the model, DESIGN.md §5):
    one unit ~ 1 ms at 2 micro-batches per stage; the split head is what the model said it would be worth."""
    pm = _pipeline_model()
    measured_fused = {2: ([15, 13], 232.0), 4: ([8, 8, 8, 4], 267.0), 8: ([4, 4, 4, 4, 4, 4, 3, 1], 309.0)}
    for n, (split, ms) in measured_fused.items():
        t, ends = pm.step_time(split, 2 * n, split_head=False)
        assert abs(t - ms) / ms < 0.03, (n, t, ms)
        t_split, _ = pm.step_time(split, 2 * n, split_head=True)
        assert t_split < t
        assert len(ends) == n and max(ends) == t
    # a single stage has no bubble: the step is exactly the sum of its work
    t1, _ = pm.step_time([28], 2, split_head=True)
    assert abs(t1 - 2 * (28 * (1.0 + 1.1 + 0.95) + 3 * 2.34)) < 1e-9
    # the search never returns something worse than the byte-balanced split it starts from
    t_best, split_best = pm.best_split(4, 28, 8)
    assert sum(split_best) == 28 and t_best <= pm.step_time([8, 8, 8, 4], 8)[0] + 1e-9
