"""The Linear-kernel harness of tests/linear_cases.py, checked without a GPU: the case tables meet the exact leg's 2^24
condition for every config, the three checkers (exact, per-element bound, guard scan) pass a faithful CPU model of the
tiled GEMM, and each planted fault fails the check aimed at it."""
import pytest
import torch

from tensorlink_b200.ml import configs as C
from tests import linear_cases as L

CONFIGS = [C.QWEN25_05B, C.QWEN25_7B, C.QWEN3_8B, C.TINY_QWEN2, C.TINY_QWEN2_D128, C.TINY_QWEN3]
SMS = (114, 132)                # H100 PCIe and SXM


@pytest.mark.parametrize("cfg", CONFIGS, ids=lambda c: c.name)
def test_model_table_meets_the_exact_condition(cfg):
    cs = L.model_calls(cfg)
    assert len({c.name for c in cs}) == len(cs)
    for c in cs:
        assert c.headroom() < L.EXACT_LIMIT, c           # K*16 + |bias| + |residual| + |C0| < 2^24
        assert c.N % 8 == 0 or c.op == "gemv", c
        if c.flags & L.A_MN:
            assert c.M % 8 == 0, c
    wgrads = [c for c in cs if "head" in c.name and c.flags & L.A_MN]
    assert {c.K for c in wgrads} >= {2048, 52} and all(c.M == cfg.vocab for c in wgrads)
    assert any(c.alias and c.op == "gemm" and not c.ws_bytes for c in cs)                # prefill in place
    assert any(c.norm and c.ws_bytes for c in cs) and any(c.next_w for c in cs)


@pytest.mark.parametrize("sms", SMS)
def test_path_matrix_reaches_every_path(sms):
    cs = L.gemm_path_matrix(sms) + L.gemv_path_matrix(sms)
    assert len({c.name for c in cs}) == len(cs)
    for c in cs:
        assert c.headroom() < L.EXACT_LIMIT, c
    kernels = {k for c in cs for k, _ in L.path_of(c, sms, env={})["kernels"]}
    for bn in (32, 128):
        for a in ("false", "true"):
            for b in ("false", "true"):
                if bn == 128 or b == "false":
                    assert f"gemm_bf16_kernel<{bn}, {a}, {b}>" in kernels
    assert {"splitk_reduce_kernel", "splitk_reduce_norm_kernel", "rmsnorm_fwd_kernel"} <= kernels
    assert {f"gemv_stream_kernel<{m}>" for m in (1, 2, 3, 4)} <= kernels
    assert any(k.startswith("gemv_kernel<") for k in kernels)
    splits = {L.gemm_path(c, sms)["splits"] for c in cs if c.op == "gemm"}
    assert splits >= set(range(1, min(8, sms // 2) + 1))
    regimes = {(d["per_sm"], d["chunked"]) for c in cs if c.op == "gemv"
               for d in L.gemv_path(c, sms, env={})["chunks"] if "per_sm" in d}
    assert regimes == {(1, False), (1, True), (2, False), (2, True)}
    reg = {L.gemv_reg_params(c.M, c.N, c.K, sms)[:2] for c in L.gemv_reg_cases(sms)}
    assert {w for _, w in reg} == {1, 2, 4, 8} and {g for g, _ in reg} == {1, 2, 4}
    mma = {L.gemv_mma_applies(c, {"TL_GEMV_MMA": "1"})["x_in_stage"] for c in L.gemv_mma_cases()}
    assert mma == {False, True}


def test_workspace_too_small_takes_the_plain_path():
    c = next(c for c in L.gemm_path_matrix(132) if c.name == "gemm.split.ws_short")
    assert L.split_plan(c, 132) is None
    from dataclasses import replace
    assert L.split_plan(replace(c, ws_bytes=c.ws_bytes + 16), 132) == (4, 8)


# cases the CPU model runs: every epilogue, every major, ragged tiles, short and ragged K, SwiGLU, the fused norm
SELF = ["gemm.kk.plain.t128", "gemm.kB.bias.t128", "gemm.Ak.res.t32", "gemm.AB.res_inplace.t128", "gemm.kk.swiglu.t32",
        "gemm.kB.f32.t128", "gemm.Ak.acc_bf16.t128", "gemm.AB.acc_f32.t128", "gemm.kk.bias_res.t32", "gemm.AB.k52.acc",
        "gemm.k40.t128"]


def _case(name):
    return next(c for c in L.gemm_path_matrix(132) if c.name == name)


@pytest.mark.parametrize("leg", ["exact", "round"])
@pytest.mark.parametrize("name", SELF)
def test_cpu_model_passes(name, leg):
    r = L.check_call(_case(name), leg, L.cpu_gemm(), "cpu")
    assert not r["errors"], "\n".join(r["errors"])
    assert leg == "exact" or 0 < r["ratio"] < 1


def test_fused_norm_check_passes_the_cpu_model():
    c = L.Case("norm", "gemm", 9, 256, 200, flags=L.EPI_RESIDUAL, alias=True, norm=True, ld_pad=0)
    for leg in ("exact", "round"):
        r = L.check_call(c, leg, L.cpu_gemm(), "cpu")
        assert not r["errors"], "\n".join(r["errors"])


# fault -> (case, leg, words the failing check's message carries)
PLANTED = {
    "drop_kblock": ("gemm.k200.ragged", "exact", "exact leg"),
    "oob_store": ("gemm.kk.plain.t128", "exact", "output C: "),
    "nan_read": ("gemm.kB.bias.t128", "exact", "exact leg"),
    "stale_row": ("gemm.k200.ragged", "exact", "exact leg"),
    "truncate": ("gemm.k200.ragged", "exact", "exact leg"),
    "swap_gate_up": ("gemm.kk.swiglu.t32", "exact", "exact leg"),
    "plus2pct": ("gemm.kk.plain.t128", "round", "rounding leg"),
}


@pytest.mark.parametrize("fault", L.FAULTS)
def test_planted_fault_is_caught(fault):
    name, leg, words = PLANTED[fault]
    r = L.check_call(_case(name), leg, L.cpu_gemm(fault), "cpu")
    assert r["errors"], f"{fault} went unnoticed"
    assert any(words in e for e in r["errors"]), r["errors"]
    print(f"{fault}: caught by the {words.strip(': ')} check\n  " + r["errors"][0].splitlines()[0])


def test_failure_report_names_tile_and_coordinates():
    r = L.check_call(_case("gemm.k200.ragged"), "exact", L.cpu_gemm("drop_kblock"), "cpu")
    msg = r["errors"][0]
    assert "by 128x128 tile" in msg and "(0, 0):" in msg and "splits=1" in msg


def test_guard_scan_sees_every_pad():
    g = L.Guard(5, 24, 32, torch.bfloat16, "cpu", L.BF16_SENTINEL)
    g.t.fill_(1.0)
    assert g.outside_changed().numel() == 0
    full = g.bits.view(5 + 2 * L.PAD_ROWS, 32)
    for r, c in ((0, 0), (L.PAD_ROWS - 1, 31), (L.PAD_ROWS, 24), (L.PAD_ROWS + 4, 31), (L.PAD_ROWS + 5, 0)):
        full[r, c] = 0
        assert g.outside_changed().tolist() == [[r - L.PAD_ROWS, c]]
        full[r, c] = L.BF16_SENTINEL
    g = L.Guard(3, 65, 65, torch.bfloat16, "cpu", L.BF16_SENTINEL)          # a GEMV output pitch: odd, unaligned
    assert g.ptr % 16 == 0 and g.outside_changed().numel() == 0
    g.rows_view[2, 64] = 0
    g.bits[-1] = 0
    assert g.outside_changed().tolist() == [[2 + L.PAD_ROWS, 64]]      # (2, 64) itself is inside the matrix
