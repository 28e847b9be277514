"""Attention kernels on peaked and rising scores, checked row by row against float64.

Unit-variance q and k (the inputs of tests/test_kernels_gpu.py) leave the online-softmax bookkeeping without effect:
any max can be subtracted short of overflow, so a kernel that gets the running max, the rescale or a split merge wrong
still passes.  Here q and k follow the score patterns of tests/attn_patterns.py (sink, rising, falling, spikes at tile,
split and warp-slice edges, wide), where that bookkeeping carries the result, and every kernel x pattern pair runs:
prefill forward (mma.sync and wgmma), backward (both forms), split-KV decode (mma and simt) and the fused decode.

Poisoning: cache rows past the valid length are NaN (the kernels promise those rows "may hold anything"), outputs start
as NaN, and each batch row has its own V / dO magnitude, so rows read past one batch row's end show up in that row.

Criteria, per row (query row b, position, head; each dq row; each dk / dv key row summed over the GQA group):
  * every output is finite;
  * |kernel - float64| <= K * |bf16 oracle - float64| + FLOOR * RMS(float64 rows of that batch row).  The forward's
    bf16 oracle is O.attention_sdpa_math.  The floor covers one-hot rows, where the oracle is exact;
  * backward: the bf16 oracle is the flash backward on that oracle's bf16 output (D = rowsum(dO * O), dS and P rounded
    to bf16), in fp32.  dq and dk are small differences of large terms, and the bf16 rounding of O moves D, so each
    row also gets CANCEL * RMS(the same gradient taken over absolute values): two bf16 roundings of what cancels.
    Without it the sink pattern, whose exact dq and dk are zero, and rising dq (up to 0.3 x its RMS off in both kernel
    and oracle, independently) could not be bounded;
  * lse: |kernel - float64| <= LSE_ATOL + LSE_RTOL * |lse| (|lse| reaches 12,600 on 'rising').
Float64 references run on the GPU in torch; the project's kernels are not involved in them.

Calibrated on an H100 80GB HBM3 (400 W power limit); worst measured error / bound over the whole file:
  prefill out 0.64, split-KV decode out 0.47, fused decode out 0.46  (K = 2, FLOOR = 2e-3)
  dq 0.56, dk 0.29, dv 0.22  (K = 2, FLOOR = 2e-3, CANCEL = 8e-3)
  lse 0.24  (LSE_ATOL = 3e-5, LSE_RTOL = 3e-6)
The mma.sync and wgmma backward give the same worst rows.  The file runs in about 10 s there (216 tests).
"""
import pytest
import torch

from tests import attn_patterns as P
from tests.attn_patterns import FWD_FLOOR, FWD_K, check_rows, oracle_fwd, ref_fwd

pytestmark = pytest.mark.gpu

BWD_K, BWD_FLOOR, BWD_CANCEL = 2.0, 2e-3, 8e-3
LSE_ATOL, LSE_RTOL = 3e-5, 3e-6
NAN = float("nan")


@pytest.fixture(scope="module")
def nat():
    from tensorlink_b200 import native
    native.require_device()
    return native


# ------------------------------------------------------------------------------------------ float64 references
def ref_bwd(q, k, v, do, scale):
    """Gradients of causal GQA attention (past = 0) in float64 for the upstream gradient do [B,S,n_h,d]:
    dq [B,S,n_h,d], dk and dv [B,n_kv,S,d] (summed over each group's query heads).  Also the same products taken over
    absolute values, |P| (|dP| + |D|) and |P|^T |dO|: the size of the terms that cancel in each gradient row."""
    B, S, n_h, d = q.shape
    n_kv = k.shape[1]
    n_rep = n_h // n_kv
    qd = q.double().transpose(1, 2)
    kk, vv = k.double().repeat_interleave(n_rep, 1), v.double().repeat_interleave(n_rep, 1)
    s = (qd @ kk.transpose(2, 3)) * scale
    above = torch.arange(S, device=q.device)[None, :] > torch.arange(S, device=q.device)[:, None]
    p = torch.softmax(s.masked_fill_(above, float("-inf")), -1)
    dod = do.double().transpose(1, 2)
    dp, D = dod @ vv.transpose(2, 3), (dod * (p @ vv)).sum(-1, keepdim=True)
    ds, dsa = p * (dp - D) * scale, p * (dp.abs() + D.abs()) * scale
    group = lambda x: x.view(B, n_kv, n_rep, S, d).sum(2)
    grads = ((ds @ kk).transpose(1, 2), group(ds.transpose(2, 3) @ qd), group(p.transpose(2, 3) @ dod))
    sizes = ((dsa @ kk.abs()).transpose(1, 2), group(dsa.transpose(2, 3) @ qd.abs()), group(p.transpose(2, 3) @ dod.abs()))
    return grads, sizes


def oracle_bwd(q, k, v, do, scale):
    """The bf16 yardstick of the backward: the flash backward on the bf16 oracle's forward, in fp32 torch on the GPU.
    D = rowsum(dO * O) from the oracle's bf16 O, P from fp32 scores and lse, dS and P rounded to bf16 for their
    products, and each query head's dk / dv partial rounded to bf16 before the group sum."""
    B, S, n_h, d = q.shape
    n_kv = k.shape[1]
    n_rep = n_h // n_kv
    o = oracle_fwd(q, k, v, scale).to(q.device).float().transpose(1, 2)
    qf = q.float().transpose(1, 2)
    kk, vv = k.float().repeat_interleave(n_rep, 1), v.float().repeat_interleave(n_rep, 1)
    s = (qf @ kk.transpose(2, 3)) * scale
    above = torch.arange(S, device=q.device)[None, :] > torch.arange(S, device=q.device)[:, None]
    s.masked_fill_(above, float("-inf"))
    p = torch.exp(s - torch.logsumexp(s, -1, keepdim=True))
    dof = do.float().transpose(1, 2)
    ds = (p * (dof @ vv.transpose(2, 3) - (dof * o).sum(-1, keepdim=True)) * scale).bfloat16().float()
    group = lambda x: x.bfloat16().float().view(B, n_kv, n_rep, S, d).sum(2)
    return ((ds @ kk).bfloat16().transpose(1, 2), group(ds.transpose(2, 3) @ qf),
            group(p.bfloat16().float().transpose(2, 3) @ dof))


# ------------------------------------------------------------------------------------------ criteria
def check_lse(what, got, ref):
    assert bool(torch.isfinite(got).all()), f"{what}: non-finite lse"
    err = (got.double() - ref).abs()
    ratio = err / (LSE_ATOL + LSE_RTOL * ref.abs())
    worst = int(ratio.argmax())
    assert float(ratio.flatten()[worst]) <= 1.0, (f"{what}: lse row {worst} off by {float(err.flatten()[worst]):.3e} "
                                                  f"at |lse| {float(ref.abs().flatten()[worst]):.1f}")


def poisoned_cache(x, T_max):
    """[B, n_kv, T, d] -> [B, n_kv, T_max, d] on the GPU with NaN in rows T..T_max-1."""
    B, n_kv, T, d = x.shape
    c = torch.full((B, n_kv, T_max, d), NAN, dtype=torch.bfloat16, device="cuda")
    c[:, :, :T] = x.cuda()
    return c


# ------------------------------------------------------------------------------------------ prefill forward
PREFILL = [  # B, S, past, n_h, n_kv, d, pattern
    (2, 100, 0, 14, 2, 64, "flat"), (2, 100, 37, 14, 2, 64, "rising"), (1, 200, 300, 28, 4, 128, "rising"),
    (2, 130, 0, 32, 8, 128, "sink"), (1, 150, 37, 4, 4, 64, "falling"), (2, 70, 0, 28, 4, 128, "spike@63"),
    (1, 97, 300, 14, 2, 64, "spike@64"), (2, 129, 0, 32, 8, 128, "spike@65"), (1, 77, 37, 28, 4, 128, "spike@T-1"),
    (3, 190, 300, 14, 2, 64, "wide"), (3, 45, 37, 32, 8, 128, "rising")]


@pytest.mark.parametrize("impl", ["mma", "wgmma"])
@pytest.mark.parametrize("B,S,past,n_h,n_kv,d,pattern", PREFILL)
def test_prefill_fwd(nat, monkeypatch, impl, B, S, past, n_h, n_kv, d, pattern):
    monkeypatch.setenv("TL_ATTN_IMPL", impl)
    _prefill_case(nat, B, S, past, n_h, n_kv, d, pattern)


def test_prefill_fwd_long_wgmma(nat, monkeypatch):
    """4096 rising keys: the two-slot TMA ring runs through 64 phases, each raising the running max."""
    monkeypatch.setenv("TL_ATTN_IMPL", "wgmma")
    _prefill_case(nat, 1, 4096, 0, 2, 1, 128, "rising")


def _prefill_case(nat, B, S, past, n_h, n_kv, d, pattern):
    T, scale = past + S, d ** -0.5
    q, k = P.make_qk(pattern, B, S, T, n_h, n_kv, d, seed=11)
    v = P.make_v(B, n_kv, T, d, seed=12)
    q, k, v = q.cuda(), k.cuda(), v.cuda()
    kc, vc = poisoned_cache(k, T + P.TILE), poisoned_cache(v, T + P.TILE)
    out = torch.full((B, S, n_h * d), NAN, dtype=torch.bfloat16, device="cuda")
    lse = torch.full((B, n_h, S), NAN, dtype=torch.float32, device="cuda")
    nat.attn_prefill_fwd(q, kc, vc, out, lse, B, S, past, n_h, n_kv, d, scale)
    ref, ref_lse = ref_fwd(q, k, v, past, scale)
    check_rows(f"{pattern} out", out.view(B, S, n_h, d), ref, oracle_fwd(q, k, v, scale), FWD_K, FWD_FLOOR)
    check_lse(f"{pattern}", lse, ref_lse)


# ------------------------------------------------------------------------------------------ backward
BWD = [  # B, S, n_h, n_kv, d, pattern
    (2, 100, 14, 2, 64, "flat"), (2, 130, 28, 4, 128, "rising"), (1, 200, 32, 8, 128, "sink"),
    (2, 97, 4, 4, 64, "falling"), (1, 150, 28, 4, 128, "spike@64"), (2, 70, 14, 2, 64, "spike@63"),
    (1, 129, 32, 8, 128, "spike@T-1"), (3, 90, 14, 2, 64, "wide"), (3, 65, 28, 4, 128, "rising")]


@pytest.mark.parametrize("impl", ["mma", "wgmma"])
@pytest.mark.parametrize("B,S,n_h,n_kv,d,pattern", BWD)
def test_bwd(nat, monkeypatch, impl, B, S, n_h, n_kv, d, pattern):
    monkeypatch.setenv("TL_ATTN_IMPL", impl)
    monkeypatch.setenv("TL_ATTN_BWD", impl)
    _bwd_case(nat, B, S, n_h, n_kv, d, pattern)


def test_bwd_long_wgmma(nat, monkeypatch):
    monkeypatch.setenv("TL_ATTN_IMPL", "wgmma")
    monkeypatch.setenv("TL_ATTN_BWD", "wgmma")
    _bwd_case(nat, 1, 4096, 2, 1, 128, "rising")


def _bwd_case(nat, B, S, n_h, n_kv, d, pattern):
    scale, n_rep, T_max = d ** -0.5, n_h // n_kv, S + P.TILE
    q, k = P.make_qk(pattern, B, S, S, n_h, n_kv, d, seed=21)
    v = P.make_v(B, n_kv, S, d, seed=22)
    do = P.make_v(B, S, n_h, d, seed=23)                 # per batch row magnitudes, as V
    q, k, v, do = q.cuda(), k.cuda(), v.cuda(), do.cuda()
    kc, vc = poisoned_cache(k, T_max), poisoned_cache(v, T_max)
    out = torch.full((B, S, n_h * d), NAN, dtype=torch.bfloat16, device="cuda")
    lse = torch.full((B, n_h, S), NAN, dtype=torch.float32, device="cuda")
    nat.attn_prefill_fwd(q, kc, vc, out, lse, B, S, 0, n_h, n_kv, d, scale)
    dq = torch.full((B, S, n_h, d), NAN, dtype=torch.bfloat16, device="cuda")
    dk = torch.full((B, n_h, T_max, d), NAN, dtype=torch.bfloat16, device="cuda")   # one partial per query head
    dv = torch.full_like(dk, NAN)
    ws = torch.empty(nat.attn_bwd_ws(B, S, n_h), dtype=torch.uint8, device="cuda")
    nat.attn_bwd(q, kc, vc, out, do.reshape(B, S, n_h * d), lse, dq, dk, dv, ws, B, S, n_h, n_kv, d, scale)
    assert bool(torch.isfinite(dk[:, :, :S]).all() and torch.isfinite(dv[:, :, :S]).all())    # every slot < S written
    assert bool(torch.isnan(dk[:, :, S:]).all() and torch.isnan(dv[:, :, S:]).all())          # and none past S
    dks = dk.float().view(B, n_kv, n_rep, T_max, d).sum(2)
    dvs = dv.float().view(B, n_kv, n_rep, T_max, d).sum(2)
    refs, sizes = ref_bwd(q, k, v, do, scale)
    for name, got, ref, oracle, size in zip(("dq", "dk", "dv"), (dq, dks[:, :, :S], dvs[:, :, :S]), refs,
                                            oracle_bwd(q, k, v, do, scale), sizes):
        check_rows(f"{pattern} {name}", got, ref, oracle, BWD_K, BWD_FLOOR, size, BWD_CANCEL)


# ------------------------------------------------------------------------------------------ split-KV decode
DECODE = [  # B, kv_len, n_h, n_kv, d, pattern
    (2, 1, 14, 2, 64, "flat"), (2, 65, 28, 4, 128, "spike@64"), (2, 66, 14, 2, 64, "spike@63"),
    (1, 67, 32, 8, 128, "spike@65"), (2, 64, 28, 4, 128, "spike@50"), (1, 129, 32, 8, 128, "spike@128"),
    (2, 130, 28, 4, 128, "spike@127"), (1, 200, 14, 2, 64, "spike@129"), (2, 257, 28, 4, 128, "spike@256"),
    (1, 300, 32, 8, 128, "spike@255"), (2, 400, 4, 4, 64, "spike@257"), (2, 256, 28, 4, 128, "spike@T-1"),
    (1, 310, 14, 2, 64, "spike@305"), (2, 4096, 28, 4, 128, "rising"), (3, 257, 32, 8, 128, "rising"),
    (1, 1000, 32, 8, 128, "sink"), (2, 500, 14, 2, 64, "falling"), (1, 777, 28, 4, 128, "wide"),
    (3, 129, 4, 4, 64, "flat")]


@pytest.mark.parametrize("impl", ["mma", "simt"])
@pytest.mark.parametrize("B,kv_len,n_h,n_kv,d,pattern", DECODE)
def test_decode(nat, monkeypatch, impl, B, kv_len, n_h, n_kv, d, pattern):
    monkeypatch.setenv("TL_DECODE_ATTN", impl)
    scale, T_max = d ** -0.5, kv_len + 100
    q, k = P.make_qk(pattern, B, 1, kv_len, n_h, n_kv, d, seed=31)
    v = P.make_v(B, n_kv, kv_len, d, seed=32)
    q, k, v = q.cuda(), k.cuda(), v.cuda()
    kc, vc = poisoned_cache(k, T_max), poisoned_cache(v, T_max)
    out = torch.full((B, n_h * d), NAN, dtype=torch.bfloat16, device="cuda")
    ws = torch.empty(nat.attn_decode_ws(B, n_h, d, T_max), dtype=torch.uint8, device="cuda")
    kvl = torch.tensor([kv_len], dtype=torch.int32, device="cuda")
    nat.attn_decode_fwd(q.reshape(B, n_h * d), kc, vc, out, kvl, ws, B, n_h, n_kv, d, scale)
    ref, _ = ref_fwd(q, k, v, kv_len - 1, scale)
    check_rows(f"{pattern} out", out.view(B, 1, n_h, d), ref, oracle_fwd(q, k, v, scale), FWD_K, FWD_FLOOR)


# ------------------------------------------------------------------------------------------ fused decode
FD_T_MAX = 2048
FUSED_GEOM = [(28, 4, 128, False), (14, 2, 64, True), (32, 4, 128, True), (16, 2, 64, False)]   # n_rep 7, 7, 8, 8
FUSED_PATTERNS = ["flat", "sink", "rising", "falling", "spike@T-1", "spike@T-2", "wide"]


FUSED_CASES = [(pos, pat) for pos in (0, 1, 255, 2046, 2047) for pat in FUSED_PATTERNS if not (pos == 0 and pat == "spike@T-2")]


@pytest.mark.parametrize("pos,pattern", FUSED_CASES)
@pytest.mark.parametrize("n_h,n_kv,d,qk_norm", FUSED_GEOM)
def test_decode_fused(nat, pos, n_h, n_kv, d, qk_norm, pattern):
    """RoPE (+ q/k-norm) + append + attention over keys 0..pos at T_max = 2048 (keys past pos are NaN).  The pattern
    sits in dim d/2-1, which the kernel's RoPE barely turns.  Cached keys are scaled by the query's designed component
    after the norm; the new key (key pos: the spike of spike@T-1) gets its logit through its own value, or through
    the k-norm gain when the norm is on.  The reference attends with the rotated query and the cache that
    rope_kv_fwd produces, and the fused kernel's cache must equal that one bit for bit."""
    B, eps, scale, T = 2, 1e-6, d ** -0.5, pos + 1
    n_rep, designed, z = n_h // n_kv, P.is_designed(pattern), P.logit_pattern(pattern, pos + 1)
    qkv, qn, kn, kc0, vc0 = (t.cuda() if t is not None else None
                             for t in P.decode_inputs(pattern, B, pos, n_h, n_kv, d, qk_norm, FD_T_MAX, eps))
    ct, st = nat.rope_table(1.0 / (1e6 ** (torch.arange(0, d, 2, dtype=torch.float32) / d)).cuda(), FD_T_MAX)
    posd = torch.tensor([pos], dtype=torch.int32, device="cuda")
    kc1, vc1 = kc0.clone(), vc0.clone()
    q = torch.empty(B, n_h * d, dtype=torch.bfloat16, device="cuda")
    nat.rope_kv_fwd(qkv, q, kc1, vc1, posd, ct, st, qn, kn, eps, 1, n_h, n_kv, d)
    kc2, vc2 = kc0.clone(), vc0.clone()
    out = torch.full((B, n_h * d), NAN, dtype=torch.bfloat16, device="cuda")
    nat.attn_decode_fused(qkv, kc2, vc2, out, posd, ct, st, qn, kn, eps, B, n_h, n_kv, d, scale)
    bits = lambda t: t.view(torch.int16)                               # (NaN rows compare too)
    assert torch.equal(bits(kc1), bits(kc2)) and torch.equal(bits(vc1), bits(vc2))
    qr, k, v = q.view(B, 1, n_h, d), kc1[:, :, :T], vc1[:, :, :T]
    ref, _ = ref_fwd(qr, k, v, pos, scale)
    if designed:      # the designed logits are in place: the new key's (set through the k-norm gain) within 5%
        s = (qr.double().view(B, n_kv, n_rep, d) @ k.double().transpose(2, 3)).mean(2) * scale
        assert abs(float(s[..., pos].mean()) - z[pos].item()) <= 0.05 * abs(z[pos].item()) + 2.0
    check_rows(f"{pattern} out", out.view(B, 1, n_h, d), ref, oracle_fwd(qr, k, v, scale), FWD_K, FWD_FLOOR)
