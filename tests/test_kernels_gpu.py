"""Kernel-level parity: every C-ABI entry point vs the CPU oracle's restatement of the same HF op.

Tolerances (stated once, used below):
  * ops with a single bf16 rounding point per output (norm, rope, Linear and its epilogues, embed):
    rel-L2 <= 1e-3 against the oracle's bf16 result (north_star tolerance; measured ~1e-4: only values
    whose fp32 accumulation order straddles a bf16 rounding boundary differ, by one ulp);
  * attention: the SDPA contract leaves the rounding point of P implementation-defined (flash kernels round
    the un-normalised exp, the math path rounds the normalised probability; torch's own CPU flash kernel
    differs from the same math by 2.7e-3 on unit-variance q/k, tests/test_oracle_vs_hf.py).  So:
      (a) against exact fp32 attention on the same bf16 inputs the kernel must be no less accurate than
          the oracle's bf16 result (<= 1.25x its error);
      (b) rel-L2 <= 4e-3 against 'sdpa_math'.  The bf16 rounding of the OUTPUT alone is ~1.5e-3, so a 1e-3
          same-dtype bound is below the output quantisation, for flat and peaked softmax alike;
  * token ids: exact.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import shard_oracle as O
from tensorlink_b200.ml import configs as C

pytestmark = pytest.mark.gpu
TOL = 1e-3
TOL_ATTN = 4e-3


@pytest.fixture(scope="module")
def nat():
    from tensorlink_b200 import native
    native.require_device()
    return native


def rnd(*shape, seed=0, std=1.0, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * std).to(dtype)


def dev(t):
    return t.cuda() if t is not None else None


@pytest.mark.parametrize("rows,H", [(1, 896), (7, 3584), (300, 4096), (5, 128), (33, 256), (2, 8192)])
def test_rmsnorm(nat, rows, H):
    x, w = rnd(rows, H, seed=1, std=2.0), (1 + 0.1 * torch.randn(H)).bfloat16()
    ref = O.rmsnorm(x, w, 1e-6)
    rstd = torch.empty(rows, dtype=torch.float32, device="cuda")
    got = nat.rmsnorm_fwd(dev(x), dev(w), 1e-6, rstd=rstd).cpu()
    assert O.rel_l2(got, ref) <= TOL
    assert (got != ref).float().mean() < 0.01
    ref_rstd = torch.rsqrt(x.float().pow(2).mean(-1) + 1e-6)
    assert torch.allclose(rstd.cpu(), ref_rstd, rtol=1e-5)


def test_embed(nat):
    table = rnd(1000, 896, seed=2)
    ids = torch.randint(0, 1000, (3, 17))
    got = nat.embed_fwd(dev(ids), dev(table)).cpu()
    assert torch.equal(got, F.embedding(ids, table))


GEMM_SHAPES = [(128, 128, 64), (128, 256, 128), (200, 264, 136), (1, 128, 64), (77, 1152, 896), (513, 896, 4864),
               (1024, 2048, 512), (300, 4608, 3584), (4096, 1024, 256)]


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_gemm_plain_and_bias(nat, M, N, K):
    a, w, b = rnd(M, K, seed=3), rnd(N, K, seed=4, std=0.05), rnd(N, seed=5, std=0.5)
    got = nat.gemm(dev(a), dev(w)).cpu()
    assert O.rel_l2(got, F.linear(a, w)) <= TOL
    got = nat.gemm(dev(a), dev(w), bias=dev(b)).cpu()
    assert O.rel_l2(got, F.linear(a, w, b)) <= TOL


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (200, 264, 136), (513, 896, 4864)])
def test_gemm_f32_out_exactness(nat, M, N, K):
    a, w = rnd(M, K, seed=3), rnd(N, K, seed=4, std=0.05)
    got = nat.gemm(dev(a), dev(w), flags=nat.EPI_OUT_F32).cpu()
    ref = a.double() @ w.double().t()
    assert O.rel_l2(got, ref) <= 1e-5


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (333, 896, 896), (64, 3584, 512)])
def test_gemm_residual(nat, M, N, K):
    a, w, r = rnd(M, K, seed=6), rnd(N, K, seed=7, std=0.05), rnd(M, N, seed=8)
    got = nat.gemm(dev(a), dev(w), residual=dev(r)).cpu()
    assert O.rel_l2(got, r + F.linear(a, w)) <= TOL


@pytest.mark.parametrize("M,I,K", [(128, 64, 64), (150, 768, 256), (96, 4864, 896)])
def test_gemm_swiglu(nat, M, I, K):
    x, wg, wu = rnd(M, K, seed=9), rnd(I, K, seed=10, std=0.08), rnd(I, K, seed=11, std=0.08)
    wgu = torch.stack([wg, wu], dim=1).reshape(2 * I, K).contiguous()      # rows 2j = gate_j, 2j+1 = up_j
    got = nat.gemm(dev(x), dev(wgu), flags=nat.EPI_SWIGLU).cpu()
    ref = F.silu(F.linear(x, wg)) * F.linear(x, wu)
    assert got.shape == (M, I)
    assert O.rel_l2(got, ref) <= TOL


def test_gemm_accumulate(nat):
    a, w = rnd(256, 128, seed=12), rnd(384, 128, seed=13, std=0.1)
    c0 = rnd(256, 384, seed=14)
    c = dev(c0.clone())
    nat.gemm(dev(a), dev(w), out=c, flags=nat.EPI_ACCUM)
    assert O.rel_l2(c.cpu(), c0 + F.linear(a, w)) <= TOL


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 384, 192), (200, 264, 136), (1024, 896, 4864)])
def test_gemm_mn_major_operands(nat, M, N, K):
    """dgrad (B given as [K,N]) and wgrad (A as [K,M], B as [K,N]) layouts without explicit transposes."""
    a, w = rnd(M, K, seed=15), rnd(N, K, seed=16, std=0.05)
    ref = (a.double() @ w.double().t())
    got = nat.gemm(dev(a), dev(w.t().contiguous()), flags=nat.B_MN_MAJOR | nat.EPI_OUT_F32, N=N).cpu()
    assert O.rel_l2(got, ref) <= 1e-5, "B MN-major"
    if M % 8 == 0:
        got = nat.gemm(dev(a.t().contiguous()), dev(w), flags=nat.A_MN_MAJOR | nat.EPI_OUT_F32, M=M, K=K).cpu()
        assert O.rel_l2(got, ref) <= 1e-5, "A MN-major"
        got = nat.gemm(dev(a.t().contiguous()), dev(w.t().contiguous()),
                       flags=nat.A_MN_MAJOR | nat.B_MN_MAJOR | nat.EPI_OUT_F32, M=M, K=K, N=N).cpu()
        assert O.rel_l2(got, ref) <= 1e-5, "A and B MN-major"


@pytest.mark.parametrize("M,N,K", [(2048, 2560, 320), (2050, 2568, 200), (4096, 4864, 896), (2304, 2304, 64)])
def test_gemm_2cta_tiles(nat, M, N, K):
    """Training-sized shapes (hundreds of 128x128 tiles, ragged edges): all epilogues and majors."""
    a, w = rnd(M, K, seed=31), rnd(N, K, seed=32, std=0.05)
    b, r = rnd(N, seed=33, std=0.5), rnd(M, N, seed=34)
    ref = a.double() @ w.double().t()
    got = nat.gemm(dev(a), dev(w), flags=nat.EPI_OUT_F32).cpu()
    assert O.rel_l2(got, ref) <= 1e-5
    assert O.rel_l2(nat.gemm(dev(a), dev(w), bias=dev(b), residual=dev(r)).cpu(), r + F.linear(a, w, b)) <= TOL
    got = nat.gemm(dev(a), dev(w.t().contiguous()), flags=nat.B_MN_MAJOR | nat.EPI_OUT_F32, N=N).cpu()
    assert O.rel_l2(got, ref) <= 1e-5, "B MN-major"
    if M % 8 == 0:
        got = nat.gemm(dev(a.t().contiguous()), dev(w.t().contiguous()),
                       flags=nat.A_MN_MAJOR | nat.B_MN_MAJOR | nat.EPI_OUT_F32, M=M, K=K, N=N).cpu()
        assert O.rel_l2(got, ref) <= 1e-5, "A and B MN-major"
        c0 = rnd(M, N, seed=35)
        c = dev(c0.clone())
        nat.gemm(dev(a.t().contiguous()), dev(w), out=c, flags=nat.A_MN_MAJOR | nat.EPI_ACCUM, M=M, K=K)
        assert O.rel_l2(c.cpu(), c0 + F.linear(a, w)) <= TOL
    if N % 16 == 0:
        got = nat.gemm(dev(a), dev(w), flags=nat.EPI_SWIGLU).cpu()
        y = F.linear(a, w)
        assert O.rel_l2(got, F.silu(y[:, 0::2]) * y[:, 1::2]) <= TOL


@pytest.mark.parametrize("M,N,K", [(32, 3584, 18944), (9, 4608, 3584), (100, 896, 4864), (32, 2048, 512)])
def test_gemm_small_m_streaming_tiles(nat, M, N, K):
    """batched-decode shapes (M <= 128, few column tiles): 32-wide tiles so every SM streams weights"""
    a, w, b, r = rnd(M, K, seed=36), rnd(N, K, seed=37, std=0.05), rnd(N, seed=38, std=0.5), rnd(M, N, seed=39)
    assert O.rel_l2(nat.gemm(dev(a), dev(w), bias=dev(b), residual=dev(r)).cpu(), r + F.linear(a, w, b)) <= TOL
    got = nat.gemm(dev(a), dev(w), flags=nat.EPI_OUT_F32).cpu()
    assert O.rel_l2(got, a.double() @ w.double().t()) <= 1e-4          # fp32 accumulation over K up to 18944
    if N % 16 == 0:
        y = F.linear(a, w)
        assert O.rel_l2(nat.gemm(dev(a), dev(w), flags=nat.EPI_SWIGLU).cpu(), F.silu(y[:, 0::2]) * y[:, 1::2]) <= TOL
    # split-K path (workspace given): same results
    ws = torch.empty(nat.gemm_splitk_ws(M, N), dtype=torch.uint8, device="cuda")
    assert O.rel_l2(nat.gemm(dev(a), dev(w), bias=dev(b), residual=dev(r), ws=ws).cpu(), r + F.linear(a, w, b)) <= TOL
    xr = dev(r.clone())
    nat.gemm(dev(a), dev(w), out=xr, residual=xr, ws=ws)                # in-place residual, as the decode layer uses it
    assert O.rel_l2(xr.cpu(), r + F.linear(a, w)) <= TOL
    assert O.rel_l2(nat.gemm(dev(a), dev(w), flags=nat.EPI_OUT_F32, ws=ws).cpu(), a.double() @ w.double().t()) <= 1e-4
    if N % 16 == 0:
        assert O.rel_l2(nat.gemm(dev(a), dev(w), flags=nat.EPI_SWIGLU, ws=ws).cpu(), F.silu(y[:, 0::2]) * y[:, 1::2]) <= TOL


GEMV_SHAPES = [(1, 1152, 896), (1, 896, 4864), (2, 4608, 3584), (3, 896, 896), (4, 3584, 18944), (8, 1024, 512),
               (1, 130, 264), (5, 2048, 1024)]


@pytest.mark.parametrize("M,N,K", GEMV_SHAPES)
def test_gemv_bias_residual(nat, M, N, K):
    x, w, b, r = rnd(M, K, seed=17), rnd(N, K, seed=18, std=0.05), rnd(N, seed=19, std=0.5), rnd(M, N, seed=20)
    assert O.rel_l2(nat.gemv(dev(x), dev(w)).cpu(), F.linear(x, w)) <= TOL
    assert O.rel_l2(nat.gemv(dev(x), dev(w), bias=dev(b)).cpu(), F.linear(x, w, b)) <= TOL
    assert O.rel_l2(nat.gemv(dev(x), dev(w), residual=dev(r)).cpu(), r + F.linear(x, w)) <= TOL


@pytest.mark.parametrize("M", [2, 3, 5, 8])
@pytest.mark.parametrize("N,K,norm,mode", [(4608, 3584, True, "bias"), (3584, 18944, False, "res"), (896, 4864, False, "res"),
                                           (9728, 896, True, "swiglu"), (37888, 3584, True, "swiglu"), (1152, 896, False, "plain")])
@pytest.mark.parametrize("mma", ["0", "1"])
def test_gemv_tensor_core_rows_2_to_8(nat, monkeypatch, mma, M, N, K, norm, mode):
    """2..8 rows: the CUDA-core stream kernel (default) and the opt-in mma.sync kernel (TL_GEMV_MMA=1: resident x, or
    x chunks streamed when K is too large) against the same oracle."""
    monkeypatch.setenv("TL_GEMV_MMA", mma)
    x, w = rnd(M, K, seed=41, std=2.0 if norm else 1.0), rnd(N, K, seed=42, std=0.05)
    g = (1 + 0.1 * torch.randn(K)).bfloat16() if norm else None
    h = O.rmsnorm(x, g, 1e-6) if norm else x
    if mode == "bias":
        b = rnd(N, seed=43, std=0.5)
        got, ref = nat.gemv(dev(x), dev(w), bias=dev(b), norm_w=dev(g), eps=1e-6), F.linear(h, w, b)
    elif mode == "res":
        r = rnd(M, N, seed=44)
        rd = dev(r.clone())
        got, ref = nat.gemv(dev(x), dev(w), out=rd, residual=rd, norm_w=dev(g), eps=1e-6), r + F.linear(h, w)
    elif mode == "swiglu":
        y = F.linear(h, w)
        got, ref = nat.gemv(dev(x), dev(w), norm_w=dev(g), eps=1e-6, flags=nat.EPI_SWIGLU), F.silu(y[:, 0::2]) * y[:, 1::2]
    else:
        got, ref = nat.gemv(dev(x), dev(w)), F.linear(h, w)
    assert O.rel_l2(got.cpu(), ref) <= TOL


@pytest.mark.parametrize("M,N,K", [(1, 1152, 896), (2, 4608, 3584), (4, 512, 256)])
def test_gemv_norm_prologue(nat, M, N, K):
    x, w, b = rnd(M, K, seed=21, std=3.0), rnd(N, K, seed=22, std=0.05), rnd(N, seed=23, std=0.5)
    g = (1 + 0.1 * torch.randn(K)).bfloat16()
    ref = F.linear(O.rmsnorm(x, g, 1e-6), w, b)
    got = nat.gemv(dev(x), dev(w), bias=dev(b), norm_w=dev(g), eps=1e-6).cpu()
    assert O.rel_l2(got, ref) <= TOL


@pytest.mark.parametrize("M,I,K", [(1, 4864, 896), (2, 768, 256), (4, 18944, 3584)])
def test_gemv_swiglu(nat, M, I, K):
    x, wg, wu = rnd(M, K, seed=24), rnd(I, K, seed=25, std=0.08), rnd(I, K, seed=26, std=0.08)
    g = (1 + 0.1 * torch.randn(K)).bfloat16()
    wgu = torch.stack([wg, wu], dim=1).reshape(2 * I, K).contiguous()
    h = O.rmsnorm(x, g, 1e-6)
    ref = F.silu(F.linear(h, wg)) * F.linear(h, wu)
    got = nat.gemv(dev(x), dev(wgu), norm_w=dev(g), eps=1e-6, flags=nat.EPI_SWIGLU).cpu()
    assert O.rel_l2(got, ref) <= TOL


@pytest.mark.parametrize("cfg", [C.TINY_QWEN2, C.TINY_QWEN2_D128, C.TINY_QWEN3], ids=lambda c: c.name)
@pytest.mark.parametrize("B,S,past", [(2, 24, 0), (1, 1, 77), (3, 5, 100)])
def test_rope_kv(nat, cfg, B, S, past):
    d, n_h, n_kv = cfg.head_dim, cfg.n_heads, cfg.n_kv_heads
    T_max = 256
    qkv = rnd(B * S, cfg.qkv_dim, seed=27)
    qn = (1 + 0.1 * torch.randn(d)).bfloat16() if cfg.qk_norm else None
    kn = (1 + 0.1 * torch.randn(d)).bfloat16() if cfg.qk_norm else None
    q, k, v = qkv.view(B, S, -1).split([cfg.q_dim, cfg.kv_dim, cfg.kv_dim], dim=-1)
    q, k, v = q.reshape(B, S, n_h, d), k.reshape(B, S, n_kv, d), v.reshape(B, S, n_kv, d)
    if cfg.qk_norm:
        q, k = O.rmsnorm(q, qn, cfg.rms_eps), O.rmsnorm(k, kn, cfg.rms_eps)
    pos = torch.arange(past, past + S)[None].expand(B, -1)
    cos, sin = O.rope_tables(cfg, pos, torch.bfloat16)
    qr, kr = O.apply_rope(q.transpose(1, 2), k.transpose(1, 2), cos, sin)
    inv = O.rope_inv_freq(cfg).cuda()
    ct, st = nat.rope_table(inv, T_max)
    ref_cos = O.rope_tables(cfg, torch.arange(T_max)[None], torch.bfloat16)[0][0, :, : d // 2]
    assert (ct.cpu() != ref_cos).float().mean() < 2e-3          # cosf vs CPU cos, after bf16 rounding
    q_out = torch.empty(B * S, cfg.q_dim, dtype=torch.bfloat16, device="cuda")
    kc = torch.zeros(B, n_kv, T_max, d, dtype=torch.bfloat16, device="cuda")
    vc = torch.zeros_like(kc)
    pos0 = torch.tensor([past], dtype=torch.int32, device="cuda")
    nat.rope_kv_fwd(dev(qkv), q_out, kc, vc, pos0, ct, st, dev(qn), dev(kn), cfg.rms_eps, S, n_h, n_kv, d)
    assert O.rel_l2(q_out.cpu().view(B, S, n_h, d).transpose(1, 2), qr) <= TOL
    assert O.rel_l2(kc.cpu()[:, :, past:past + S], kr) <= TOL
    assert torch.equal(vc.cpu()[:, :, past:past + S], v.transpose(1, 2))
    assert kc.cpu()[:, :, :past].abs().sum() == 0 and kc.cpu()[:, :, past + S:].abs().sum() == 0


def _attn_case(B, S, past, n_h, n_kv, d, seed, std=1.0):
    T = past + S
    q = rnd(B, S, n_h, d, seed=seed, std=std)
    k = rnd(B, n_kv, T, d, seed=seed + 1, std=std)
    v = rnd(B, n_kv, T, d, seed=seed + 2)
    ref = O.attention_sdpa_math(q.transpose(1, 2), k, v, d ** -0.5, n_h // n_kv)
    kk, vv = O.repeat_kv(k, n_h // n_kv).float(), O.repeat_kv(v, n_h // n_kv).float()
    s = (q.transpose(1, 2).float() @ kk.transpose(2, 3)) * d ** -0.5 + O.causal_mask(S, T, torch.float32)
    f32 = (F.softmax(s, -1) @ vv).transpose(1, 2).reshape(B, S, -1)
    return q, k, v, ref, f32


@pytest.mark.parametrize("impl", ["mma", "wgmma"])
@pytest.mark.parametrize("B,S,past,n_h,n_kv,d", [(2, 100, 0, 4, 2, 64), (1, 64, 0, 14, 2, 64), (1, 50, 37, 4, 2, 128),
                                                 (2, 257, 0, 8, 2, 128), (1, 1, 200, 4, 4, 64), (1, 130, 300, 7, 1, 128),
                                                 (1, 512, 0, 28, 4, 128), (2, 300, 100, 14, 2, 64), (1, 1024, 0, 4, 2, 128),
                                                 (1, 192, 0, 28, 4, 128), (2, 65, 63, 8, 1, 64), (1, 129, 0, 12, 2, 128),
                                                 (3, 31, 0, 4, 4, 64), (1, 640, 0, 16, 2, 128), (2, 96, 160, 6, 3, 64),
                                                 (1, 256, 256, 32, 8, 128), (1, 384, 0, 14, 2, 64), (2, 200, 8, 4, 1, 128)])
def test_attn_prefill(nat, monkeypatch, impl, B, S, past, n_h, n_kv, d):
    """Both prefill kernels, each forced for every case: mma.sync tiles (attention.cu) and the wgmma kernel
    (attention_wgmma.cu); sequence lengths on and off the 64-row tile grid, with and without a cached prefix, GQA groups
    1..8, both head sizes."""
    monkeypatch.setenv("TL_ATTN_IMPL", impl)
    q, k, v, ref, f32 = _attn_case(B, S, past, n_h, n_kv, d, seed=30)
    T_max = past + S + 19
    kc = torch.zeros(B, n_kv, T_max, d, dtype=torch.bfloat16)
    vc = torch.zeros_like(kc)
    kc[:, :, :past + S], vc[:, :, :past + S] = k, v
    kc[:, :, past + S:], vc[:, :, past + S:] = 40.0, -30.0      # poison: keys beyond the valid length must be ignored
    out = torch.empty(B, S, n_h * d, dtype=torch.bfloat16, device="cuda")
    lse = torch.empty(B, n_h, S, dtype=torch.float32, device="cuda")
    nat.attn_prefill_fwd(dev(q), dev(kc), dev(vc), out, lse, B, S, past, n_h, n_kv, d, d ** -0.5)
    got = out.cpu()
    assert O.rel_l2(got, f32) <= 1.25 * O.rel_l2(ref, f32) + 1e-4
    assert O.rel_l2(got, ref) <= TOL_ATTN
    kk = O.repeat_kv(k, n_h // n_kv).float()
    s = (q.transpose(1, 2).float() @ kk.transpose(2, 3)) * d ** -0.5 + O.causal_mask(S, past + S, torch.float32)
    assert torch.allclose(lse.cpu(), torch.logsumexp(s, -1), rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("B,kv_len,n_h,n_kv,d", [(1, 1, 14, 2, 64), (2, 127, 4, 2, 128), (1, 128, 28, 4, 128),
                                                 (3, 129, 8, 8, 64), (1, 1000, 28, 4, 128), (2, 2048, 32, 8, 128),
                                                 (32, 4096, 28, 4, 128), (4, 65, 16, 2, 128), (5, 193, 28, 4, 128)])
@pytest.mark.parametrize("impl", ["mma", "simt"])
def test_attn_decode(nat, B, kv_len, n_h, n_kv, d, impl, monkeypatch):
    """split-KV decode attention: the tensor-core split kernel (default: the GQA group's query heads are the MMA's M rows)
    and the CUDA-core one (TL_DECODE_ATTN=simt) against the oracle."""
    monkeypatch.setenv("TL_DECODE_ATTN", impl)
    q, k, v, ref, f32 = _attn_case(B, 1, kv_len - 1, n_h, n_kv, d, seed=40)
    T_max = kv_len + 100
    kc = torch.zeros(B, n_kv, T_max, d, dtype=torch.bfloat16)
    vc = torch.zeros_like(kc)
    kc[:, :, :kv_len], vc[:, :, :kv_len] = k, v
    kc[:, :, kv_len:] = 50.0        # poison: keys beyond kv_len must be ignored
    out = torch.empty(B, n_h * d, dtype=torch.bfloat16, device="cuda")
    ws = torch.empty(nat.attn_decode_ws(B, n_h, d, T_max), dtype=torch.uint8, device="cuda")
    kvl = torch.tensor([kv_len], dtype=torch.int32, device="cuda")
    nat.attn_decode_fwd(dev(q.reshape(B, n_h * d)), dev(kc), dev(vc), out, kvl, ws, B, n_h, n_kv, d, d ** -0.5)
    got = out.cpu().view(B, 1, -1)
    assert O.rel_l2(got, f32) <= 1.25 * O.rel_l2(ref, f32) + 1e-4
    assert O.rel_l2(got, ref) <= TOL_ATTN


@pytest.mark.parametrize("cfg", [C.TINY_QWEN2, C.TINY_QWEN2_D128, C.TINY_QWEN3], ids=lambda c: c.name)
@pytest.mark.parametrize("B,past", [(1, 0), (2, 1), (1, 127), (3, 128), (1, 700)])
def test_attn_decode_fused_equals_unfused(nat, cfg, B, past):
    """Fused RoPE + append + attention == rope_kv_fwd -> attn_decode_fwd (same rounding points): outputs within one
    bf16 ulp-level reordering, cache contents identical; and both satisfy the oracle bound."""
    d, n_h, n_kv = cfg.head_dim, cfg.n_heads, cfg.n_kv_heads
    T_max = past + 9
    qkv = rnd(B, cfg.qkv_dim, seed=70).cuda()
    qn = dev((1 + 0.1 * torch.randn(d)).bfloat16()) if cfg.qk_norm else None
    kn = dev((1 + 0.1 * torch.randn(d)).bfloat16()) if cfg.qk_norm else None
    kc0 = rnd(B, n_kv, T_max, d, seed=71).cuda()
    vc0 = rnd(B, n_kv, T_max, d, seed=72).cuda()
    ct, st = nat.rope_table(O.rope_inv_freq(cfg).cuda(), T_max)
    pos = torch.tensor([past], dtype=torch.int32, device="cuda")
    kvl = torch.tensor([past + 1], dtype=torch.int32, device="cuda")
    kc1, vc1 = kc0.clone(), vc0.clone()
    q = torch.empty(B, cfg.q_dim, dtype=torch.bfloat16, device="cuda")
    ref = torch.empty(B, cfg.q_dim, dtype=torch.bfloat16, device="cuda")
    nat.rope_kv_fwd(qkv, q, kc1, vc1, pos, ct, st, qn, kn, cfg.rms_eps, 1, n_h, n_kv, d)
    ws = torch.empty(nat.attn_decode_ws(B, n_h, d, T_max), dtype=torch.uint8, device="cuda")
    nat.attn_decode_fwd(q, kc1, vc1, ref, kvl, ws, B, n_h, n_kv, d, d ** -0.5)
    kc2, vc2 = kc0.clone(), vc0.clone()
    got = torch.empty_like(ref)
    nat.attn_decode_fused(qkv, kc2, vc2, got, pos, ct, st, qn, kn, cfg.rms_eps, B, n_h, n_kv, d, d ** -0.5)
    assert torch.equal(kc1, kc2) and torch.equal(vc1, vc2)
    assert O.rel_l2(got.cpu(), ref.cpu()) <= TOL_ATTN      # two valid P-rounding orders (global vs per-split max)
    # oracle: attention of the rotated query over keys 0..past
    qr = q.cpu().view(B, 1, n_h, d)
    o_ref = O.attention_sdpa_math(qr.transpose(1, 2), kc1.cpu()[:, :, :past + 1], vc1.cpu()[:, :, :past + 1], d ** -0.5,
                                  n_h // n_kv)
    assert O.rel_l2(got.cpu().view(B, 1, -1), o_ref) <= TOL_ATTN


@pytest.mark.parametrize("M,V,H", [(1, 1024, 256), (2, 151936, 896), (4, 2048, 512)])
def test_lmhead_argmax(nat, M, V, H):
    x, w = rnd(M, H, seed=50, std=2.0), rnd(V, H, seed=51, std=0.05)
    g = (1 + 0.1 * torch.randn(H)).bfloat16()
    ref_logits = F.linear(O.rmsnorm(x, g, 1e-6), w)
    ids = torch.empty(M, dtype=torch.int64, device="cuda")
    logits = torch.empty(M, V, dtype=torch.bfloat16, device="cuda")
    ws = torch.empty(nat.lmhead_ws(M, V), dtype=torch.uint8, device="cuda")
    nat.lmhead_argmax(dev(x), dev(w), dev(g), 1e-6, ids, logits, ws)
    assert O.rel_l2(logits.cpu(), ref_logits) <= TOL
    # ids must be the argmax of the logits the kernel itself produced (first index on ties) ...
    assert torch.equal(ids.cpu(), logits.cpu().float().argmax(-1))
    # ... and equal the oracle's wherever the oracle's top-2 margin exceeds one bf16 ulp of the top value
    top2 = ref_logits.float().topk(2, -1).values
    safe = (top2[:, 0] - top2[:, 1]) > top2[:, 0].abs() * 2 ** -7
    assert torch.equal(ids.cpu()[safe], ref_logits.float().argmax(-1)[safe])


def test_argmax_ties_pick_lowest_index(nat):
    logits = torch.full((3, 5000), -1.0).bfloat16()
    logits[0, [4999, 17, 3000]] = 2.0
    logits[1, [4098, 4097]] = 0.5
    logits[2, :] = 1.0
    ids = torch.empty(3, dtype=torch.int64, device="cuda")
    ws = torch.empty(3 * 64 * 8, dtype=torch.uint8, device="cuda")
    nat.argmax_bf16(dev(logits), ids, ws)
    assert ids.cpu().tolist() == [17, 4097, 0]


# ------------------------------------------------------------------------------------------ peer-memory mailbox
def test_peer_wait_signal_put(nat):
    """A waiter on one stream is released by a put on another: payload first, then the sequence number (csrc/peer.cu);
    counters advance on the device; a wait nobody answers gives up after its timeout and raises the error word."""
    import time
    ptr, handle = nat.peer_alloc(8192)
    assert len(handle) == 64
    raw = nat.tensor_from_ptr(ptr, 8192)
    assert raw.data_ptr() == ptr and int(raw.sum()) == 0
    flag, buf = raw[:4].view(torch.int32), raw[256:256 + 2048].view(torch.bfloat16)
    want, sent, err = (torch.zeros(1, dtype=torch.int32, device="cuda") for _ in range(3))
    wait_ns = torch.zeros(1, dtype=torch.int64, device="cuda")
    # first use of each kernel sequentially: lazy module loading synchronises the context, which must not happen while
    # a waiter is already spinning (the pipeline loads them when it instantiates its graphs, before any traffic)
    nat.peer_put(buf, rnd(1024, seed=69).cuda(), flag, sent)
    nat.peer_wait(flag, want, err, wait_ns)
    bump = torch.zeros(2, dtype=torch.int32, device="cuda")
    nat.peer_signal(flag, sent, bump=bump[0:1])             # the optional bookkeeping counters advance with the handshake
    nat.peer_wait(flag, want, err, wait_ns, bump=bump[1:2])
    torch.cuda.synchronize()
    assert int(want) == 2 and int(sent) == 2 and int(flag) == 2 and int(err) == 0 and bump.tolist() == [1, 1]
    wait_ns.zero_()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    for rnd_i in range(3):
        src = rnd(1024, seed=70 + rnd_i).cuda()
        out = torch.empty(1024, dtype=torch.bfloat16, device="cuda")
        torch.cuda.synchronize()
        with torch.cuda.stream(s1):
            nat.peer_wait(flag, want, err, wait_ns)
            out.copy_(buf)
        time.sleep(0.02)
        with torch.cuda.stream(s2):
            nat.peer_put(buf, src, flag, sent)
        torch.cuda.synchronize()
        assert int(err) == 0
        assert torch.equal(out, src)
        assert int(want) == rnd_i + 3 and int(sent) == rnd_i + 3 and int(flag) == rnd_i + 3
    assert int(wait_ns) > 3 * 5_000_000          # the three waits really waited (>= 3 x 20 ms sleeps, generous margin)
    nat.peer_wait(flag, want, err, None, timeout_ns=3_000_000)   # nobody signals 5: times out after 3 ms
    torch.cuda.synchronize()
    assert int(err) == 1
    del raw, flag, buf
    nat.peer_free(ptr)


@pytest.mark.parametrize("M,N,K,mode", [(32, 3584, 3584, "res"), (8, 896, 4864, "res"), (5, 4608, 3584, "bias"), (16, 512, 256, "res"),
                                        (200, 1024, 2048, "res")])
def test_gemm_with_fused_following_rmsnorm(nat, M, N, K, mode):
    """tl_gemm_bf16_ws_norm: C as tl_gemm_bf16_ws, plus H = RMSNorm(C) * g — fused into the split-K reduce (decode shapes)
    or a separate launch (no split / M > 128); C is identical, H equals tl_rmsnorm_fwd(C) up to the reduction order."""
    a, w = rnd(M, K, seed=51), rnd(N, K, seed=52, std=0.05)
    g = (1 + 0.1 * torch.randn(N)).bfloat16()
    ws = torch.empty(nat.gemm_splitk_ws(min(M, 128), N), dtype=torch.uint8, device="cuda")
    kw = dict(bias=dev(rnd(N, seed=53, std=0.5))) if mode == "bias" else dict(residual=dev(rnd(M, N, seed=54)))
    c_ref = nat.gemm(dev(a), dev(w), ws=ws, **kw)
    h_ref = nat.rmsnorm_fwd(c_ref, dev(g), 1e-6)
    h = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    c = nat.gemm(dev(a), dev(w), ws=ws, norm_w=dev(g), eps=1e-6, h_out=h, **kw)
    assert torch.equal(c, c_ref) and O.rel_l2(h.cpu(), h_ref.cpu()) <= 1e-4      # (sum of squares reduced in another order)
    ref = F.linear(a, w, kw.get("bias").cpu() if mode == "bias" else None)
    if mode == "res":
        ref = kw["residual"].cpu() + ref
    assert O.rel_l2(c.cpu(), ref) <= TOL and O.rel_l2(h.cpu(), O.rmsnorm(ref, g, 1e-6)) <= 2 * TOL
