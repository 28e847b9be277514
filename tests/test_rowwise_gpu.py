"""The row-wise and element-wise kernels element by element (tests/rowwise_cases.py): SwiGLU over every finite bf16 gate,
RMSNorm, the rotary tables, RoPE + KV append and its backward, cross-entropy's dlogits, the embedding gather, the gradient
commits, the AdamW step (both TL_ADAM_STREAM settings) and the two samplers draw by draw.  Every output sits between
sentinel guards and every input between NaN guards.  Each test prints its measured worst |err| / bound and flip count."""
import json
import os
import subprocess
import sys

import pytest
import torch

from tests import rowwise_cases as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
_TABLES = {}


@pytest.fixture(scope="module")
def launch():
    from tensorlink_b200 import native
    native.require_device()
    return R.NativeLaunch(native)


def tables(launch, d, theta=1e6, max_pos=1024):
    if (d, theta) not in _TABLES:
        _TABLES[(d, theta)] = launch.rope_table(R.hf_inv_freq(d, theta).cuda(), max_pos)
    return _TABLES[(d, theta)]


def _ok(r, what):
    assert not r["errors"], r["errors"][:6]
    print(f"ROWWISE {what}: " + ", ".join(f"{k}={v}" for k, v in r.items() if k not in ("errors", "tables")))


@pytest.mark.parametrize("c", R.swiglu_cases(), ids=lambda c: c.name)
def test_swiglu_every_gate(launch, c):
    """forward: torch's bf16 F.silu(g)*u except where silu lies within 2^-20 of a tie (g <= -89 included: -0);
    backward: the float64 autograd chain, exact outside its band"""
    r = R.run_swiglu(c, launch, DEV)
    _ok(r, f"swiglu[{c.name}]")
    if c.ups:
        assert r["low_gates_exact"] > 0


@pytest.mark.parametrize("H", R.NORM_H)
def test_rmsnorm_fwd(launch, H):
    """exact outside a 2^-16 tie band of x·rstd; rstd within 2^-21; zero rows and fp32-overflowing rows as HF"""
    _ok(R.run_rmsnorm(H, launch, DEV), f"rmsnorm[H={H}]")


def test_rmsnorm_rejects_wide_rows(launch):
    with pytest.raises(RuntimeError, match="8192"):
        R.run_rmsnorm(8200, launch, DEV)


@pytest.mark.parametrize("d,theta", [(64, 1e6), (128, 1e6), (64, 1e4), (128, 1e4)])
def test_rope_table(launch, d, theta):
    """HF's fp32 inv_freq·pos -> cos / sin -> bf16 at every position up to 32,768: exact outside a 2^-21 band"""
    r = R.run_rope_table(d, theta, 32768, launch, DEV)
    _ok(r, f"rope_table[d={d},theta={theta:g}]")


@pytest.mark.parametrize("c", R.rope_fwd_cases(), ids=lambda c: c.name)
def test_rope_kv_fwd(launch, c):
    """HF's bf16 apply_rotary_pos_emb bit for bit on the kernel's own tables (q/k-norm: the 2^-16 band); V copied exactly;
    cache slots outside [pos0, pos0+S) untouched"""
    _ok(R.run_rope_fwd(c, tables(launch, c.d), launch, DEV), f"rope_fwd[{c.name}]")


@pytest.mark.parametrize("leg", ["exact", "round"])
@pytest.mark.parametrize("c", R.rope_bwd_cases(), ids=lambda c: c.name)
def test_rope_kv_bwd(launch, c, leg):
    """exact leg: integer partials, equal to the float64 value rounded once; rounding leg: one bf16 ulp + 2^-20 of the
    summed magnitudes; the NaN rows S..T_max-1 of dk / dv never reach the output"""
    _ok(R.run_rope_bwd(c, leg, tables(launch, c.d), launch, DEV), f"rope_bwd[{c.name}/{leg}]")


@pytest.mark.parametrize("c", R.ce_cases(), ids=lambda c: c.name)
def test_ce_dlogits(launch, c):
    """(softmax - onehot)·scale per element within one bf16 ulp + 2^-20·p_max·scale (+ 2^-126·scale); in place equals
    out of place bit for bit; ignored rows exactly 0"""
    _ok(R.run_ce(c, launch, DEV), f"ce[{c.name}]")


@pytest.mark.parametrize("H", [8, 896, 3584])
@pytest.mark.parametrize("n", [1, 31, 33, 4100])
def test_embed_fwd(launch, H, n):
    """an exact copy; ids < 0 or >= vocab give row 0"""
    _ok(R.run_embed(H, n, launch, DEV), f"embed[H={H},n={n}]")


@pytest.mark.parametrize("kind", ["add", "scale_bf16", "scale_f32", "f32_to_bf16", "alias"])
def test_gradient_commits(launch, kind):
    """bit for bit against the stated rounding points: fp32 s·b + a (one rounding), then bf16; accumulate both ways;
    the aliased scale_add(x, x, s, accumulate=False) of commit_head"""
    ns = R.COMMIT_N + (R.COMMIT_N_RAGGED if kind in ("scale_f32", "f32_to_bf16") else ())
    accs = (False,) if kind in ("add", "alias") else (False, True)
    for n in ns:
        for acc in accs:
            _ok(R.run_commit(kind, n, acc, launch, DEV), f"{kind}[n={n},acc={acc}]")


def test_bf16_commits_reject_ragged_sizes(launch):
    a = torch.zeros(12, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(RuntimeError, match="n % 8"):
        launch.add_inplace(a, a.clone())
    with pytest.raises(RuntimeError, match="n % 8"):
        launch.scale_add(a, a.clone(), 0.5)


@pytest.mark.parametrize("a", R.ADAM_CFGS, ids=lambda a: a.name)
@pytest.mark.parametrize("n", R.ADAM_N)
def test_adamw_one_step(launch, n, a):
    """per step from the kernel's own state: m, v within 4 fp32 ulp; p within one bf16 ulp, exact outside the 2^-16 band;
    sentinels past n"""
    _ok(R.run_adam(n, a, R.ADAM_STEPS, launch, DEV), f"adam[{a.name},n={n}]")


def test_adamw_stage_spans_zero_grad_and_lr0(launch):
    spans, n = R.stage_adam_spans([4096, 130, 70000, 896], 4099)
    for a in R.ADAM_CFGS:
        _ok(R.run_adam(n, a, (1, 2, 10, 1000), launch, DEV, spans=spans), f"adam[{a.name},spans]")
        _ok(R.run_adam(4099, a, (1, 10), launch, DEV, zero_grad=True), f"adam[{a.name},zero_grad]")
        _ok(R.run_adam(4099, a, (5,), launch, DEV, lr_zero=True), f"adam[{a.name},lr0]")


def test_adamw_plain_loads_in_a_fresh_process(tmp_path):
    """TL_ADAM_STREAM=0 (plain loads and stores, read once per process) passes the same checks"""
    out = tmp_path / "adam.json"
    env = dict(os.environ, PYTHONPATH=ROOT, TL_ADAM_STREAM="0")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "rowwise_env_worker.py"), str(out)], env=env,
                       capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(out.read_text())
    assert not res["errors"], res["errors"][:6]
    assert res["cases"] >= 18
    print(f"ROWWISE adam[TL_ADAM_STREAM=0]: ratio_p={res['ratio_p']}, ratio_mv={res['ratio_mv']}")


@pytest.mark.parametrize("c", R.sample_cases(), ids=lambda c: c.name)
def test_sample_draw_by_draw(launch, c):
    """every draw equals the Philox + float64 inverse-CDF model's token unless its target lies in the derived error band
    of a CDF boundary; fewer than 0.1 % of draws land there"""
    r = R.run_sample(c, launch, DEV)
    _ok(r, f"sample[{c.name}]")
    assert r["band"] < 1e-3 * r["draws"], r
