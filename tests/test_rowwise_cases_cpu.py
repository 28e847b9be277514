"""The row-wise harness of tests/rowwise_cases.py, checked without a GPU: the Philox model reproduces Random123's
known-answer vectors, every checker passes a CPU model of the kernels written with their rounding points, the sampling
cases pin their kept sets and keep the band share under 0.1 %, and each planted fault fails the check aimed at it."""
import numpy as np
import pytest
import torch

from tests import rowwise_cases as R

DEV = "cpu"
TABLES = {}


def tables(d, max_pos=1024):
    if d not in TABLES:
        TABLES[d] = R.CpuKernels().rope_table(R.hf_inv_freq(d, 1e6), max_pos)
    return TABLES[d]


def test_philox_known_answers():
    for ctr, key, want in R.PHILOX_KAT:
        got = R.philox4x32_10(tuple(np.array([c], np.uint64) for c in ctr), key)
        assert [int(x[0]) for x in got] == list(want)
    u = R.philox_u(R.SEED, 3, np.arange(100000, dtype=np.uint64))
    assert u.min() >= 0 and u.max() < 1 and abs(u.mean() - 0.5) < 0.005


def test_bf16_rounding_helpers():
    x = torch.tensor([1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, -(1.0 + 2 ** -8), 3.0e38, 3.4e38, 2 ** -134, 0.0, -0.0],
                     dtype=torch.float64)
    assert torch.equal(R.bits(R.rbf(x)), x.float().to(torch.bfloat16).view(torch.int16))
    r = torch.randn(100000, dtype=torch.float64) * 10.0 ** torch.randint(-30, 30, (100000,))
    assert torch.equal(R.bits(R.rbf(r.float().double())), r.float().to(torch.bfloat16).view(torch.int16))
    near, other, tie = R.neighbours(torch.tensor([1.0 + 2 ** -8], dtype=torch.float64))
    assert float(tie[0]) == 0 and {float(near[0]), float(other[0])} == {1.0, 1.0 + 2 ** -7}


@pytest.mark.parametrize("c", [R.swiglu_cases()[0], R.swiglu_cases()[-1]], ids=lambda c: c.name)
def test_swiglu_model_passes(c):
    r = R.run_swiglu(c, R.CpuKernels(), DEV)
    assert not r["errors"], r["errors"]
    if c.ups:
        assert r["low_gates_exact"] > 0                       # g <= -89 is in the exhaustive set and gives torch's -0


def test_swiglu_swap_is_caught():
    r = R.run_swiglu(R.swiglu_cases()[-1], R.CpuKernels("swiglu_swap"), DEV)
    assert any("d_gate" in e for e in r["errors"]) and any("d_up" in e for e in r["errors"])


@pytest.mark.parametrize("H", R.NORM_H)
def test_rmsnorm_model_passes(H):
    r = R.run_rmsnorm(H, R.CpuKernels(), DEV)
    assert not r["errors"], r["errors"]


def test_rmsnorm_rejects_wide_rows():
    with pytest.raises(RuntimeError):
        R.run_rmsnorm(8200, R.CpuKernels(), DEV)


@pytest.mark.parametrize("d,theta", [(64, 1e6), (128, 1e4)])
def test_rope_table_model_passes(d, theta):
    r = R.run_rope_table(d, theta, 4096, R.CpuKernels(), DEV)
    assert not r["errors"], r["errors"]


@pytest.mark.parametrize("c", R.rope_fwd_cases(), ids=lambda c: c.name)
def test_rope_fwd_model_passes(c):
    r = R.run_rope_fwd(c, tables(c.d), R.CpuKernels(), DEV)
    assert not r["errors"], r["errors"]


@pytest.mark.parametrize("leg", ["exact", "round"])
@pytest.mark.parametrize("c", R.rope_bwd_cases(), ids=lambda c: c.name)
def test_rope_bwd_model_passes(c, leg):
    r = R.run_rope_bwd(c, leg, tables(c.d), R.CpuKernels(), DEV)
    assert not r["errors"], r["errors"]


@pytest.mark.parametrize("fault", ["rope_nrep_minus_1", "rope_pos_off_by_one"])
def test_rope_bwd_faults_are_caught(fault):
    c = R.rope_bwd_cases()[0]
    for leg in ("exact", "round"):
        r = R.run_rope_bwd(c, leg, tables(c.d), R.CpuKernels(fault), DEV)
        assert any(f"rope_bwd[{c.name}/{leg}]" in e for e in r["errors"]), (fault, leg)


@pytest.mark.parametrize("c", R.ce_cases(), ids=lambda c: c.name)
def test_ce_model_passes(c):
    r = R.run_ce(c, R.CpuKernels(), DEV)
    assert not r["errors"], r["errors"]


def test_ce_label_off_is_caught():
    r = R.run_ce(R.ce_cases()[1], R.CpuKernels("ce_label_off"), DEV)
    assert any(".dlogits" in e for e in r["errors"])


@pytest.mark.parametrize("H,n", [(8, 1), (896, 33), (3584, 31), (8, 4100)])
def test_embed_model_passes(H, n):
    assert not R.run_embed(H, n, R.CpuKernels(), DEV)["errors"]


@pytest.mark.parametrize("kind", ["add", "scale_bf16", "scale_f32", "f32_to_bf16", "alias"])
def test_commit_model_passes(kind):
    for n in (R.COMMIT_N_RAGGED if kind in ("scale_f32", "f32_to_bf16") else R.COMMIT_N)[:3]:
        for acc in ((False,) if kind in ("alias", "add") else (False, True)):
            r = R.run_commit(kind, n, acc, R.CpuKernels(), DEV)
            assert not r["errors"], r["errors"]


def test_commit_faults_are_caught():
    assert R.run_commit("scale_bf16", 4096, False, R.CpuKernels("scale_add_ignores_acc"), DEV)["errors"]
    assert R.run_commit("alias", 4096, False, R.CpuKernels("scale_add_ignores_acc"), DEV)["errors"]
    assert R.run_commit("f32_to_bf16", 4099, False, R.CpuKernels("f32_to_bf16_trunc"), DEV)["errors"]


@pytest.mark.parametrize("a", R.ADAM_CFGS, ids=lambda a: a.name)
def test_adam_model_passes(a):
    for n in (1, 9, 4099):
        r = R.run_adam(n, a, R.ADAM_STEPS, R.CpuKernels(), DEV)
        assert not r["errors"], r["errors"]
    spans, n = R.stage_adam_spans([1000, 130, 4096], 77)
    assert not R.run_adam(n, a, (1, 2), R.CpuKernels(), DEV, spans=spans)["errors"]
    assert not R.run_adam(4099, a, (1, 10), R.CpuKernels(), DEV, zero_grad=True)["errors"]
    assert not R.run_adam(4099, a, (3,), R.CpuKernels(), DEV, lr_zero=True)["errors"]


def test_adam_tail_fault_is_caught():
    r = R.run_adam(4099, R.ADAM_CFGS[0], (1,), R.CpuKernels("adam_no_tail"), DEV)
    assert any(".p" in e for e in r["errors"]) and any(".m" in e for e in r["errors"])
    assert not R.run_adam(4096, R.ADAM_CFGS[0], (1,), R.CpuKernels("adam_no_tail"), DEV)["errors"]


@pytest.mark.parametrize("c", R.sample_cases(), ids=lambda c: c.name)
def test_sample_cases_are_pinned_and_rarely_banded(c):
    r = R.run_sample(c, R.CpuKernels(), DEV)
    assert not r["errors"], r["errors"]
    assert r["band"] < 1e-3 * r["draws"], (r["band"], r["draws"])


def test_sample_case_features():
    cs = R.sample_cases()
    assert {c.V for c in cs} >= {1, 7, 48, 1000, 151936} and max(c.M for c in cs) == 9
    assert {c.temperature for c in cs} >= {0.05, 1.0, 20.0}
    assert any(c.top_k == 1 for c in cs) and any(c.tie_k for c in cs) and any(c.top_k >= c.V for c in cs)
    assert any(c.proc and c.n_ban >= c.V for c in cs) and any(c.proc and c.penalty != 1 and 0 < c.n_ban < c.V for c in cs)
    c = next(c for c in cs if c.tie_k)
    logits = R.sample_inputs(c)[0]
    for m in range(c.M):
        rm = R.sample_row_model(logits[m], c.temperature, c.top_k, c.top_p)
        assert rm.kept.sum() > c.top_k                     # the whole tie group at the k-th value is kept


@pytest.mark.parametrize("fault,case", [("next_token", "V48.t20"), ("top_p_low", "V48.p")])
def test_sampler_faults_are_caught(fault, case):
    c = next(c for c in R.sample_cases() if c.name == case)
    r = R.run_sample(c, R.CpuKernels(fault), DEV)
    assert any("draws differ" in e for e in r["errors"]), r["errors"]
