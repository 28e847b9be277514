"""The Linear kernels element by element (tests/linear_cases.py): an exact leg on integer operands (bit for bit), a
rounding leg on realistic operands (a per-element bound), guard bands around every operand and output, and proof from
torch.profiler that each case ran the kernels the host dispatch should pick on this device's SM count.  Covers the path
matrix (operand majors x epilogues x tile widths, split-K at every split count, the GEMV regimes and its fallback), every
Linear call of the model for six configs, the L2-prefetch hint, the settings read once per process, and the argument
checks."""
import json
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import pytest
import torch

from tensorlink_b200.ml import configs as C
from tests import linear_cases as L

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def nat():
    from tensorlink_b200 import native
    native.require_device()
    return native


@pytest.fixture(scope="module")
def sms(nat):
    return torch.cuda.get_device_properties(0).multi_processor_count


def family(c, sms):
    if c.op == "gemv":
        return "gemv.norm" if c.norm else "gemv"
    if c.norm:
        return "gemm.fused_norm"
    if L.split_plan(c, sms):
        return "gemm.split_k"
    return "gemm.f32" if c.f32 else "gemm.bf16"


def run(nat, sms, cases, legs=("exact", "round"), env=None):
    """every case on every leg under one profiler session; fails with every wrong element, guard and path found"""
    launch = L.native_launch(nat)
    errors, expected, ratios = [], [], {}
    with L.KernelLog() as log:
        for c in cases:
            for leg in legs:
                if leg == "exact" and not c.exact_ok:
                    continue
                r = L.check_call(c, leg, launch, "cuda", sms, env)
                errors += r["errors"]
                expected.append((f"{c.name}/{leg}", r["path"]["kernels"]))
                if leg == "round":
                    f = family(c, sms)
                    ratios[f] = max(ratios.get(f, 0.0), r["ratio"])
        torch.cuda.synchronize()
    path_error = L.match_paths(expected, log.kernels, log.all_names)
    print("worst |err| / bound:", {k: round(v, 3) for k, v in sorted(ratios.items())})
    print("kernels:", sorted({k for k, _ in log.kernels}))
    assert not errors, "\n".join(errors[:20]) + (f"\n... {len(errors)} failures" if len(errors) > 20 else "")
    assert not path_error, path_error
    return ratios


def test_gemm_path_matrix(nat, sms):
    run(nat, sms, L.gemm_path_matrix(sms))


def test_gemv_path_matrix(nat, sms):
    run(nat, sms, L.gemv_path_matrix(sms))


def test_gemv_mma_opt_in(nat, sms, monkeypatch):
    """TL_GEMV_MMA is read on every call: the mma.sync kernel with resident and with streamed x"""
    monkeypatch.setenv("TL_GEMV_MMA", "1")
    run(nat, sms, L.gemv_mma_cases(), env=dict(os.environ))


@pytest.mark.parametrize("cfg", [C.QWEN25_05B, C.QWEN25_7B, C.QWEN3_8B, C.TINY_QWEN2, C.TINY_QWEN2_D128, C.TINY_QWEN3],
                         ids=lambda c: c.name)
def test_model_calls(nat, sms, cfg):
    cases = L.model_calls(cfg)
    run(nat, sms, cases)


@pytest.mark.parametrize("leg", ["exact", "round"])
def test_gemv_next_w_changes_no_bit(nat, sms, leg):
    """tl_gemv_bf16_pf's L2 prefetch of the next weight is a hint only: the same bits as tl_gemv_bf16"""
    from dataclasses import replace
    launch = L.native_launch(nat)
    cases = [c for c in L.gemv_path_matrix(sms) if c.M in (1, 3, 5) and (leg == "round" or c.exact_ok)]
    for c in cases:
        a = L.check_call(c, leg, launch, "cuda", sms, want_bits=True)
        b = L.check_call(replace(c, next_w=True), leg, launch, "cuda", sms, want_bits=True)
        assert not a["errors"] and not b["errors"], a["errors"] + b["errors"]
        assert a["bits_c"] == b["bits_c"], c.name


def test_fused_norm_leaves_c_as_the_unfused_call(nat, sms):
    """C of tl_gemm_bf16_ws_norm equals C of tl_gemm_bf16_ws bit for bit on the fused split-K reduce and on the plain
    path followed by rmsnorm_fwd; H is checked element by element in the path matrix"""
    from dataclasses import replace
    launch = L.native_launch(nat)
    cases = [c for c in L.gemm_path_matrix(sms) if c.norm]
    assert {L.gemm_path(c, sms)["kernels"][-1][0] for c in cases} >= {"splitk_reduce_norm_kernel", "rmsnorm_fwd_kernel"}
    for leg in ("exact", "round"):
        for c in cases:
            a = L.check_call(c, leg, launch, "cuda", sms, want_bits=True)
            b = L.check_call(replace(c, norm=False), leg, launch, "cuda", sms, want_bits=True)
            assert not a["errors"] and not b["errors"], a["errors"] + b["errors"]
            assert a["bits_c"] == b["bits_c"], (c.name, leg)


# ------------------------------------------------------------------------------------------------ once-read settings
SETTINGS = {"default": {}, "reg": {"TL_GEMV_IMPL": "reg"}, "ctas1": {"TL_GEMV_CTAS_PER_SM": "1"},
            "ctas2": {"TL_GEMV_CTAS_PER_SM": "2"}, "ring110": {"TL_GEMV_RING_KB": "110"}, "nopdl": {"TL_PDL": "0"}}
ONCE_READ = ("TL_GEMV_IMPL", "TL_GEMV_CTAS_PER_SM", "TL_GEMV_RING_KB", "TL_PDL", "TL_GEMV_MMA")


def test_settings_read_once_give_the_same_bits(tmp_path):
    """each setting in a fresh process: both legs pass, the recorded kernels are the ones the setting selects, and the
    exact leg gives the default's bits"""
    base = {k: v for k, v in os.environ.items() if k not in ONCE_READ}

    def one(name):              # subprocess.run kills the worker if it outlives its timeout
        return subprocess.run([sys.executable, os.path.join(ROOT, "tests", "linear_env_worker.py"), str(tmp_path / f"{name}.json")],
                              env=dict(base, PYTHONPATH=ROOT, **SETTINGS[name]), capture_output=True, text=True, timeout=300,
                              cwd=ROOT)

    with ThreadPoolExecutor(len(SETTINGS)) as ex:       # the workers are independent: start-up dominates, so overlap it
        runs = dict(zip(SETTINGS, ex.map(one, SETTINGS)))
    results = {}
    for name, r in runs.items():
        assert r.returncode == 0, (name, r.stderr[-3000:])
        res = json.loads((tmp_path / f"{name}.json").read_text())
        assert not res["errors"], (name, res["errors"][:10])
        assert not res["path_error"], (name, res["path_error"])
        print(name, "kernels:", res["n_kernels"], "worst |err| / bound:", res["ratios"])
        results[name] = res
    ref = results["default"]["bits"]
    for name, res in results.items():
        diff = [k for k, v in res["bits"].items() if k.endswith("/exact") and v != ref[k]]
        assert not diff, (name, diff[:10])


# ------------------------------------------------------------------------------------------------ argument checks
BF = torch.bfloat16


class ArgBufs:
    """operands, output and workspace sized for the largest arguments below, all holding a sentinel"""

    def __init__(self):
        self.a = L.Guard(256, 2048, 2048, BF, "cuda", L.BF16_SENTINEL)
        self.b = L.Guard(512, 2048, 2048, BF, "cuda", L.BF16_SENTINEL)
        self.c = L.Guard(256, 1024, 1024, torch.float32, "cuda", L.F32_SENTINEL)
        self.v = L.Guard(256, 1024, 1024, BF, "cuda", L.BF16_SENTINEL)     # residual or norm gain
        self.h = L.Guard(256, 1024, 1024, BF, "cuda", L.BF16_SENTINEL)
        self.ws = L.Guard(1, 8 * 128 * 512, 8 * 128 * 512, torch.float32, "cuda", L.F32_SENTINEL)
        self.all = [self.a, self.b, self.c, self.v, self.h, self.ws]
        self.snaps = [g.snapshot() for g in self.all]

    def unchanged(self):
        torch.cuda.synchronize()
        return all(torch.equal(g.bits, s) for g, s in zip(self.all, self.snaps))


SW, RES, F32, ACC, BIAS = L.EPI_SWIGLU, L.EPI_RESIDUAL, L.EPI_OUT_F32, L.EPI_ACCUM, L.EPI_BIAS
# name -> (M, N, K, ldc or None (= output width), flags); M = 16, N = 256, K = 2048 takes the split-K path when a
# workspace is given, so the checks are made on that path too
GEMM_REJECTS = {
    "n_mod8": (16, 252, 2048, None, 0),
    "k_mod8_kmajor": (16, 256, 2044, None, 0),
    "k_mod8_a_kmajor": (16, 256, 2044, None, L.B_MN),
    "swiglu_residual": (16, 256, 2048, None, SW | RES),
    "swiglu_f32": (16, 256, 2048, None, SW | F32),
    "swiglu_accum": (16, 256, 2048, None, SW | ACC),
    "swiglu_n_mod16": (16, 264, 2048, None, SW),
    "ldc_small": (16, 256, 2048, 248, 0),
    "ldc_unaligned": (16, 256, 2048, 260, 0),
    "a_mn_m_mod8": (12, 256, 2048, None, L.A_MN),
    "bias_null": (16, 256, 2048, None, BIAS),
}


@pytest.mark.parametrize("entry", ["gemm", "gemm_ws", "gemm_ws_norm"])
@pytest.mark.parametrize("case", sorted(GEMM_REJECTS))
def test_gemm_argument_checks(nat, case, entry):
    M, N, K, ldc, flags = GEMM_REJECTS[case]
    g = ArgBufs()
    lib = nat.load()
    c_cols = N // 2 if flags & SW else N
    ldc = c_cols if ldc is None else ldc
    lda = M if flags & L.A_MN else K
    ldb = N if flags & L.B_MN else K
    res = g.v.ptr if flags & RES else None
    bias = None                                     # BIAS without a pointer is one of the cases; others never set it
    st = nat._stream()
    if entry == "gemm":
        rc = lib.tl_gemm_bf16(g.a.ptr, g.b.ptr, g.c.ptr, M, N, K, lda, ldb, ldc, bias, res, flags, st)
    elif entry == "gemm_ws":
        rc = lib.tl_gemm_bf16_ws(g.a.ptr, g.b.ptr, g.c.ptr, M, N, K, lda, ldb, ldc, bias, res, flags, g.ws.ptr,
                                 g.ws.cols * 4, st)
    else:
        rc = lib.tl_gemm_bf16_ws_norm(g.a.ptr, g.b.ptr, g.c.ptr, M, N, K, lda, ldb, ldc, bias, res, flags, g.ws.ptr,
                                      g.ws.cols * 4, g.v.ptr, L.EPS, g.h.ptr, st)
    with pytest.raises(nat.NativeError):
        nat._check(rc, f"{entry}:{case}")
    assert g.unchanged(), f"{entry}:{case} wrote memory before rejecting its arguments"


def test_gemm_split_path_still_runs_with_valid_arguments(nat, sms):
    """the shape of the argument checks above does take the split-K path when its arguments are valid"""
    c = L.Case("argshape", "gemm", 16, 256, 2048, flags=RES, ws_bytes=L.splitk_ws(16, 256), ld_pad=0)
    assert L.split_plan(c, sms)
    run(nat, sms, [c], legs=("exact",))


@pytest.mark.parametrize("case", ["m9", "swiglu_residual", "norm_fused_ldc", "norm_wide"])
def test_gemv_and_norm_argument_checks(nat, case):
    g = ArgBufs()
    lib = nat.load()
    st = nat._stream()
    if case == "m9":
        rc = lib.tl_gemv_bf16_pf(g.a.ptr, g.b.ptr, g.c.ptr, 9, 256, 512, None, None, None, L.EPS, 0, None, 0, st)
    elif case == "swiglu_residual":
        rc = lib.tl_gemv_bf16_pf(g.a.ptr, g.b.ptr, g.c.ptr, 2, 256, 512, None, g.v.ptr, None, L.EPS, SW | RES, None, 0, st)
    elif case == "norm_wide":   # neither norm pass takes rows wider than 8192: rejected before C is written
        rc = lib.tl_gemm_bf16_ws_norm(g.a.ptr, g.b.ptr, g.c.ptr, 16, 8320, 64, 64, 64, 8320, None, None, 0, g.ws.ptr,
                                      g.ws.cols * 4, g.v.ptr, L.EPS, g.h.ptr, st)
    else:       # the fused norm writes H with pitch N: C must have it too
        rc = lib.tl_gemm_bf16_ws_norm(g.a.ptr, g.b.ptr, g.c.ptr, 16, 256, 2048, 2048, 2048, 264, None, None, 0, g.ws.ptr,
                                      g.ws.cols * 4, g.v.ptr, L.EPS, g.h.ptr, st)
    with pytest.raises(nat.NativeError):
        nat._check(rc, case)
    assert g.unchanged(), f"{case} wrote memory before rejecting its arguments"
