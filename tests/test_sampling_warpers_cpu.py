"""generate's min_p / typical_p / epsilon_cutoff / eta_cutoff on the host: keyword parsing into the sampling dict, and
the float64 row model of the device rule (tests/warpers_model.py) against HF's own warper chain on fp32 copies, with
planted faults that each check must catch."""
import numpy as np
import pytest
import torch

from tensorlink_b200.ml import DistributedModel
from tensorlink_b200.ml import configs as C
from tensorlink_b200.ml import module as M
from tensorlink_b200.p2p.link import StageLink
from tests.oracle_stage import OracleStage
from tests.warpers_model import FAULTS, Warp, hf_warped, processed_values, replay_kept_weight, warped_model

CFG = C.TINY_QWEN2


class _Sampler(OracleStage):
    def set_sampling(self, sampling):
        pass


@pytest.fixture(scope="module")
def dm():
    return DistributedModel(CFG, training=False, max_batch=4, max_seq=64, _stage_factory=_Sampler, device="cpu",
                            link=StageLink(0, 1))


def _sampling(dm, **kw):
    req, _ = dm._request(torch.zeros(1, 4, dtype=torch.int64), dict(kw))
    return req.sampling


def test_neutral_values_leave_sampling_unchanged(dm):
    base = _sampling(dm, do_sample=True, seed=3)
    for kw in (dict(min_p=None), dict(min_p=0.0), dict(typical_p=None), dict(typical_p=1.0), dict(typical_p=1.5),
               dict(epsilon_cutoff=None), dict(epsilon_cutoff=0.0), dict(epsilon_cutoff=1.0), dict(epsilon_cutoff=-0.5),
               dict(eta_cutoff=None), dict(eta_cutoff=0.0), dict(eta_cutoff=2.0),
               dict(min_p=0, typical_p=1, epsilon_cutoff=0, eta_cutoff=0)):
        assert _sampling(dm, do_sample=True, seed=3, **kw) == base, kw


def test_active_values_enter_sampling(dm):
    s = _sampling(dm, do_sample=True, seed=3, min_p=0.1, typical_p=0.9, epsilon_cutoff=3e-4, eta_cutoff=1e-3)
    assert s["min_p"] == 0.1 and s["typical_p"] == 0.9 and s["epsilon"] == 3e-4 and s["eta"] == 1e-3
    assert _sampling(dm, do_sample=True, seed=3, min_p=1)["min_p"] == 1.0


def test_hf_value_errors(dm):
    from transformers.generation import logits_process as L
    for kw, hf in ((dict(min_p=-0.1), lambda: L.MinPLogitsWarper(-0.1)), (dict(min_p=1.5), lambda: L.MinPLogitsWarper(1.5)),
                   (dict(typical_p=0.0), lambda: L.TypicalLogitsWarper(0.0)),
                   (dict(typical_p=-1.0), lambda: L.TypicalLogitsWarper(-1.0))):
        with pytest.raises(ValueError):
            hf()
        with pytest.raises(ValueError):
            _sampling(dm, do_sample=True, **kw)


def test_greedy_ignores_the_warpers(dm):
    for kw in (dict(min_p=0.5), dict(min_p=7.0), dict(typical_p=-1.0), dict(epsilon_cutoff=0.2), dict(eta_cutoff=0.3)):
        assert _sampling(dm, **kw) is None
        assert _sampling(dm, do_sample=False, **kw) is None


def test_top_h_still_raises(dm):
    for kw in (dict(do_sample=True, top_h=0.4), dict(top_h=0.4)):
        with pytest.raises(NotImplementedError):
            _sampling(dm, **kw)


# ------------------------------------------------------------------------------------------------ the row model vs HF
VS = (7, 48, 1000, 151_936)
TS = (0.05, 0.7, 1.0, 20.0)
ALONE = {"min_p": Warp(min_p=0.08), "typical": Warp(typical_p=0.6), "epsilon": Warp(epsilon=3e-3),
         "eta": Warp(eta=2e-3)}
CHAIN = Warp(min_p=0.02, typical_p=0.9, epsilon=1e-4, eta=3e-4)
PAIR = Warp(min_p=0.1, epsilon=0.03)             # epsilon right after a min_p that removes real mass
PAIR_ETA = Warp(min_p=0.02, eta=0.01)            # eta on a set whose entropy is far from the whole row's


def _row(V, seed, ties=False):
    g = torch.Generator().manual_seed(seed)
    if ties:                                      # few distinct values: a tie group at every boundary
        x = torch.randint(-12, 9, (V,), generator=g).float() / 3
    else:
        x = torch.randn(V, generator=g) * 2.5
    return x.to(torch.bfloat16)


def _proc_inputs(V, seed):
    g = torch.Generator().manual_seed(seed + 7)
    present = (torch.rand(V, generator=g) < 0.2).numpy()
    return present, 1.3


def _cases():
    out = []
    for V in VS:
        for T in TS:
            for name, w in list(ALONE.items()) + [("chain", CHAIN), ("min_p_eps", PAIR), ("min_p_eta", PAIR_ETA)]:
                tk, tp = (40, 0.95) if name == "chain" else (0, 1.0)
                for proc in (False, True):
                    for ties in ((False, True) if V <= 1000 else (False,)):
                        out.append((V, T, name, w, tk, tp, proc, ties))
    return out


def _compare(case, fault=None):
    """(pinned, agree) of the model (with a planted fault) against HF's chain on one row"""
    V, T, name, w, tk, tp, proc, ties = case
    seed = V * 31 + int(T * 100) + len(name) + 1000 * proc + 7 * ties
    row = _row(V, seed, ties)
    present, pen = _proc_inputs(V, seed) if proc else (None, 1.0)
    rm = warped_model(row, T, tk, tp, w, proc=proc, present=present, penalty=pen, fault=fault)
    x = processed_values(row, present, None, pen) if proc else row.float().numpy()
    xs = torch.from_numpy(np.ascontiguousarray(x))[None]
    hf = torch.isfinite(hf_warped(xs, T, tk, tp, w))[0].numpy()
    pinned = rm.pinned
    if tp < 1.0:
        # HF's TopP cuts a tie group at its boundary by sort position, where the device keeps the whole group: such a
        # row says nothing about the stages after it
        before = warped_model(row, T, tk, tp, Warp(), proc=proc, present=present, penalty=pen)
        pinned &= bool(np.array_equal(before.kept, torch.isfinite(hf_warped(xs, T, tk, tp, Warp()))[0].numpy()))
    return pinned, bool(np.array_equal(rm.kept, hf))


def test_row_model_agrees_with_hf():
    bad, pinned, n = [], 0, 0
    for case in _cases():
        p, ok = _compare(case)
        n += 1
        pinned += p
        if p and not ok:
            bad.append(case[:3] + case[6:])
    assert not bad, bad[:8]
    assert pinned >= 0.6 * n, (pinned, n)


@pytest.mark.parametrize("fault", [f for f in FAULTS if f != "kept_weight_no_hi"])
def test_planted_faults_fail(fault):
    target = {"min_p_extra_bin": ("min_p", "chain"), "typical_shift": ("typical", "chain"),
              "eps_before_min_p": ("min_p_eps",), "eta_whole_row": ("min_p_eta",)}[fault]
    caught = 0
    for case in _cases():
        if case[2] not in target:
            continue
        p, ok = _compare(case, fault)
        caught += p and not ok
    assert caught > 0, fault


def _typical_drops_argmax():
    # one dominant token far above a large, flat band: the band holds the mean, so typical keeps it without the top
    x = torch.full((48,), 0.0)
    x[0] = 6.0
    x[1:21] = 3.0
    return x.to(torch.bfloat16)


def test_typical_drops_the_argmax():
    row = _typical_drops_argmax()
    w = Warp(typical_p=0.3)
    rm = warped_model(row, 1.0, 0, 1.0, w)
    hf = torch.isfinite(hf_warped(row.float()[None], 1.0, 0, 1.0, w))[0].numpy()
    assert rm.pinned and np.array_equal(rm.kept, hf)
    assert not rm.kept[0] and rm.kept[1:21].all() and not rm.kept[21:].any()
    assert rm.w[1] == 1.0                             # rebased on the kept top: the kept mass cannot round to zero


def test_min_p_one_keeps_the_top_tie_group():
    row = torch.tensor([1.0, 3.0, 3.0, 2.9, -1.0], dtype=torch.bfloat16)
    rm = warped_model(row, 0.7, 0, 1.0, Warp(min_p=1.0))
    assert rm.kept.tolist() == [False, True, True, False, False]


def test_kept_weight_ignoring_hi_fails():
    row = _typical_drops_argmax()
    rm = warped_model(row, 1.0, 0, 1.0, Warp(typical_p=0.3))
    s = row.float().numpy().astype(np.float64)
    good, bad = replay_kept_weight(rm, s), replay_kept_weight(rm, s, "kept_weight_no_hi")
    assert np.array_equal(good > 0, rm.kept)
    assert not np.array_equal(bad > 0, rm.kept) and bad[0] > 0
