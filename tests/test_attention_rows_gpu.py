"""The left-padded (`_rows`) attention and RoPE entry points, row by row against float64.

Row b of a batch starts with kv_start[b] pad slots: its keys are the cache slots kv_start[b].. and its RoPE positions
start at its first real token.  Every batch below mixes distinct starts at tile (64), split (128 / 256) and warp-slice
edges, including 0 and the last slot (one real token).  Cache slots below each start and past the valid length are
NaN, and outputs start as NaN, so a kernel that reads a pad slot, or lets it reach P·V, fails on that row.

Each real query row must meet the per-row bound of tests/test_attention_numerics_gpu.py (2 x the bf16 oracle's error
+ 2e-3 x RMS, against float64 over keys [kv_start, pos]); a pad query row must be exactly 0 with lse = -inf.  With
every start at 0 each `_rows` entry point must equal its existing twin bit for bit, and the RoPE / cache append of a
padded row must equal the plain kernel on the same row unpadded at positions 0..L-1.
"""
import pytest
import torch

from tests import attn_patterns as P
from tests.test_attention_numerics_gpu import FWD_FLOOR, FWD_K, NAN, check_lse, check_rows, oracle_fwd, ref_fwd

pytestmark = pytest.mark.gpu

GEOMS = [(14, 2, 64), (28, 4, 128), (32, 8, 128)]
PATTERNS = ["flat", "rising", "sink"]          # sink: key 0 of each row's real keys, i.e. its first valid (mid-tile) key


@pytest.fixture(scope="module")
def nat():
    from tensorlink_b200 import native
    native.require_device()
    return native


def _starts(T):
    """Distinct starts at tile, split and warp-slice edges, and T-1 (one real key); all below T."""
    base = [0, 1, 63, 64, 65, 255, 256, 257, T - 1]
    out = []
    for s in base:
        if s < T and s not in out:
            out.append(s)
    return out


def _padded_cache(rows, T_max):
    """rows: per batch row (start, [n_kv, L, d] bf16) -> [B, n_kv, T_max, d] with NaN outside [start, start + L)."""
    n_kv, _, d = rows[0][1].shape
    c = torch.full((len(rows), n_kv, T_max, d), NAN, dtype=torch.bfloat16, device="cuda")
    for b, (s, x) in enumerate(rows):
        c[b, :, s:s + x.shape[1]] = x.cuda()
    return c


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


# ------------------------------------------------------------------------------------------ prefill
@pytest.mark.parametrize("impl", ["mma", "wgmma"])
@pytest.mark.parametrize("past", [0, 37])
@pytest.mark.parametrize("n_h,n_kv,d", GEOMS)
@pytest.mark.parametrize("pattern", PATTERNS)
def test_prefill_rows(nat, monkeypatch, impl, past, n_h, n_kv, d, pattern):
    monkeypatch.setenv("TL_ATTN_IMPL", impl)
    S = 300
    T, scale, T_max = past + S, d ** -0.5, past + S + P.TILE
    starts = _starts(T)
    B = len(starts)
    q = torch.randn(B, S, n_h, d, generator=torch.Generator().manual_seed(5)).bfloat16()   # pad rows: finite noise
    krows, vrows, real = [], [], []
    for b, s in enumerate(starts):
        L = T - s                                    # real keys of row b
        Sq = min(S, L)                               # its real query rows: the last Sq
        qb, kb = P.make_qk(pattern, 1, Sq, L, n_h, n_kv, d, seed=100 + b)
        vb = P.make_v(1, n_kv, L, d, seed=200 + b) * P.BATCH_MAG[b % len(P.BATCH_MAG)]
        q[b, S - Sq:] = qb[0]
        krows.append((s, kb[0]))
        vrows.append((s, vb[0].bfloat16()))
        real.append(Sq)
    q = q.cuda()
    kc, vc = _padded_cache(krows, T_max), _padded_cache(vrows, T_max)
    ks = torch.tensor(starts, dtype=torch.int32, device="cuda")
    out = torch.full((B, S, n_h * d), NAN, dtype=torch.bfloat16, device="cuda")
    lse = torch.full((B, n_h, S), NAN, dtype=torch.float32, device="cuda")
    nat.attn_prefill_fwd(q, kc, vc, out, lse, B, S, past, n_h, n_kv, d, scale, kv_start=ks)
    for b, s in enumerate(starts):
        Sq = real[b]
        pad = S - Sq
        assert bool((out[b, :pad] == 0).all()), f"row {b} (start {s}): pad query rows not zero"
        assert bool((lse[b, :, :pad] == float("-inf")).all()), f"row {b}: pad lse not -inf"
        qb = q[b:b + 1, pad:]
        kb, vb = kc[b:b + 1, :, s:T], vc[b:b + 1, :, s:T]
        ref, ref_lse = ref_fwd(qb, kb, vb, T - s - Sq, scale)
        check_rows(f"{pattern} row {b} start {s}", out[b:b + 1, pad:].view(1, Sq, n_h, d), ref,
                   oracle_fwd(qb, kb, vb, scale), FWD_K, FWD_FLOOR)
        check_lse(f"{pattern} row {b} start {s}", lse[b:b + 1, :, pad:], ref_lse)


@pytest.mark.parametrize("impl", ["mma", "wgmma"])
@pytest.mark.parametrize("past", [0, 37])
def test_prefill_rows_zero_start_equals_plain(nat, monkeypatch, impl, past):
    monkeypatch.setenv("TL_ATTN_IMPL", impl)
    B, S, n_h, n_kv, d = 3, 150, 28, 4, 128
    T, T_max = past + S, past + S + 64
    q, k = P.make_qk("rising", B, S, T, n_h, n_kv, d, seed=3)
    v = P.make_v(B, n_kv, T, d, seed=4)
    kc, vc = _padded_cache([(0, k[b]) for b in range(B)], T_max), _padded_cache([(0, v[b]) for b in range(B)], T_max)
    q = q.cuda()
    outs = []
    for ks in (None, torch.zeros(B, dtype=torch.int32, device="cuda")):
        o = torch.full((B, S, n_h * d), NAN, dtype=torch.bfloat16, device="cuda")
        lse = torch.full((B, n_h, S), NAN, dtype=torch.float32, device="cuda")
        nat.attn_prefill_fwd(q, kc, vc, o, lse, B, S, past, n_h, n_kv, d, d ** -0.5, kv_start=ks)
        outs.append((o, lse))
    assert torch.equal(_bits(outs[0][0]), _bits(outs[1][0])) and torch.equal(_bits(outs[0][1]), _bits(outs[1][1]))


# ------------------------------------------------------------------------------------------ split-KV decode
@pytest.mark.parametrize("impl", ["mma", "simt"])
@pytest.mark.parametrize("n_h,n_kv,d", GEOMS)
@pytest.mark.parametrize("pattern", PATTERNS)
def test_decode_rows(nat, monkeypatch, impl, n_h, n_kv, d, pattern):
    monkeypatch.setenv("TL_DECODE_ATTN", impl)
    kv_len, T_max, scale = 700, 800, d ** -0.5
    starts = [0, 1, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 512, kv_len - 1]
    B = len(starts)
    q = torch.empty(B, 1, n_h, d, dtype=torch.bfloat16)
    krows, vrows = [], []
    for b, s in enumerate(starts):
        qb, kb = P.make_qk(pattern, 1, 1, kv_len - s, n_h, n_kv, d, seed=300 + b)
        q[b] = qb[0]
        krows.append((s, kb[0]))
        vrows.append((s, (P.make_v(1, n_kv, kv_len - s, d, seed=400 + b) * P.BATCH_MAG[b % 3])[0].bfloat16()))
    q = q.cuda()
    kc, vc = _padded_cache(krows, T_max), _padded_cache(vrows, T_max)
    ks = torch.tensor(starts, dtype=torch.int32, device="cuda")
    kvl = torch.tensor([kv_len], dtype=torch.int32, device="cuda")
    ws = torch.empty(nat.attn_decode_ws(B, n_h, d, T_max), dtype=torch.uint8, device="cuda")
    out = torch.full((B, n_h * d), NAN, dtype=torch.bfloat16, device="cuda")
    nat.attn_decode_fwd(q.reshape(B, n_h * d), kc, vc, out, kvl, ws, B, n_h, n_kv, d, scale, kv_start=ks)
    for b, s in enumerate(starts):
        qb, kb, vb = q[b:b + 1], kc[b:b + 1, :, s:kv_len], vc[b:b + 1, :, s:kv_len]
        ref, _ = ref_fwd(qb, kb, vb, kv_len - s - 1, scale)
        check_rows(f"{pattern} row {b} start {s}", out[b:b + 1].view(1, 1, n_h, d), ref, oracle_fwd(qb, kb, vb, scale),
                   FWD_K, FWD_FLOOR)
    # every start at 0: the _rows kernels equal the plain ones bit for bit
    kc0 = _padded_cache([(0, kc[b, :, :kv_len].nan_to_num(0.0)) for b in range(B)], T_max)
    vc0 = _padded_cache([(0, vc[b, :, :kv_len].nan_to_num(0.0)) for b in range(B)], T_max)
    o1 = torch.full_like(out, NAN)
    o2 = torch.full_like(out, NAN)
    nat.attn_decode_fwd(q.reshape(B, n_h * d), kc0, vc0, o1, kvl, ws, B, n_h, n_kv, d, scale)
    nat.attn_decode_fwd(q.reshape(B, n_h * d), kc0, vc0, o2, kvl, ws, B, n_h, n_kv, d, scale,
                        kv_start=torch.zeros(B, dtype=torch.int32, device="cuda"))
    assert torch.equal(_bits(o1), _bits(o2))


# ------------------------------------------------------------------------------------------ RoPE + cache append
def _tables(nat, d, T):
    return nat.rope_table(1.0 / (1e6 ** (torch.arange(0, d, 2, dtype=torch.float32) / d)).cuda(), T)


@pytest.mark.parametrize("n_h,n_kv,d", GEOMS)
@pytest.mark.parametrize("qk_norm", [False, True])
def test_rope_rows_equals_unpadded(nat, n_h, n_kv, d, qk_norm):
    """A padded row's q_out and cache slots equal tl_rope_kv_fwd on the same row alone at positions 0..L-1."""
    S, T_max, eps = 300, 320, 1e-6
    starts = _starts(S)
    B = len(starts)
    g = torch.Generator().manual_seed(7)
    qkv = (torch.randn(B * S, (n_h + 2 * n_kv) * d, generator=g)).bfloat16().cuda()
    qn = (1 + 0.1 * torch.randn(d, generator=g)).bfloat16().cuda() if qk_norm else None
    kn = (1 + 0.1 * torch.randn(d, generator=g)).bfloat16().cuda() if qk_norm else None
    ct, st = _tables(nat, d, T_max)
    pos0 = torch.zeros(1, dtype=torch.int32, device="cuda")
    kc = torch.full((B, n_kv, T_max, d), NAN, dtype=torch.bfloat16, device="cuda")
    vc = torch.full_like(kc, NAN)
    q = torch.full((B * S, n_h * d), NAN, dtype=torch.bfloat16, device="cuda")
    ks = torch.tensor(starts, dtype=torch.int32, device="cuda")
    nat.rope_kv_fwd(qkv, q, kc, vc, pos0, ct, st, qn, kn, eps, S, n_h, n_kv, d, kv_start=ks)
    assert bool(torch.isfinite(q).all())                     # pad tokens are rotated at position 0
    for b, s in enumerate(starts):
        L = S - s
        kc1 = torch.full((1, n_kv, T_max, d), NAN, dtype=torch.bfloat16, device="cuda")
        vc1 = torch.full_like(kc1, NAN)
        q1 = torch.empty(L, n_h * d, dtype=torch.bfloat16, device="cuda")
        nat.rope_kv_fwd(qkv[b * S + s:(b + 1) * S].contiguous(), q1, kc1, vc1, pos0, ct, st, qn, kn, eps, L, n_h, n_kv, d)
        assert torch.equal(_bits(q[b * S + s:(b + 1) * S]), _bits(q1)), f"row {b} start {s}: q_out"
        assert torch.equal(_bits(kc[b, :, s:S]), _bits(kc1[0, :, :L])), f"row {b} start {s}: k cache"
        assert torch.equal(_bits(vc[b, :, s:S]), _bits(vc1[0, :, :L])), f"row {b} start {s}: v cache"
    # all-zero starts: the plain kernel's bits
    kc2, vc2, q2 = torch.full_like(kc, NAN), torch.full_like(vc, NAN), torch.full_like(q, NAN)
    kc3, vc3, q3 = torch.full_like(kc, NAN), torch.full_like(vc, NAN), torch.full_like(q, NAN)
    nat.rope_kv_fwd(qkv, q2, kc2, vc2, pos0, ct, st, qn, kn, eps, S, n_h, n_kv, d)
    nat.rope_kv_fwd(qkv, q3, kc3, vc3, pos0, ct, st, qn, kn, eps, S, n_h, n_kv, d,
                    kv_start=torch.zeros(B, dtype=torch.int32, device="cuda"))
    assert torch.equal(_bits(q2), _bits(q3)) and torch.equal(_bits(kc2), _bits(kc3)) and torch.equal(_bits(vc2), _bits(vc3))


# ------------------------------------------------------------------------------------------ fused decode
@pytest.mark.parametrize("n_h,n_kv,d", GEOMS)
@pytest.mark.parametrize("qk_norm", [False, True])
@pytest.mark.parametrize("pattern", PATTERNS)
def test_decode_fused_rows(nat, n_h, n_kv, d, qk_norm, pattern):
    """T_max = 2048, new token at slot pos = 1500: RoPE at pos - kv_start[b], append at pos, attention over
    [kv_start[b], pos].  The cache equals tl_rope_kv_fwd_rows' (which equals the unpadded row's, test above)."""
    T_max, pos, eps, scale = 2048, 1500, 1e-6, d ** -0.5
    starts = _starts(pos + 1) + [1499]
    B = len(starts)
    g = torch.Generator().manual_seed(11)
    qkv = (torch.randn(B, (n_h + 2 * n_kv) * d, generator=g) * 0.5).bfloat16().cuda()
    qn = (1 + 0.1 * torch.randn(d, generator=g)).bfloat16().cuda() if qk_norm else None
    kn = (1 + 0.1 * torch.randn(d, generator=g)).bfloat16().cuda() if qk_norm else None
    krows, vrows = [], []
    for b, s in enumerate(starts):
        _, kb = P.make_qk(pattern, 1, 1, pos - s, n_h, n_kv, d, seed=500 + b) if pos > s else (None, None)
        if kb is None:
            kb = torch.empty(1, n_kv, 0, d, dtype=torch.bfloat16)
        krows.append((s, kb[0]))
        vrows.append((s, (P.make_v(1, n_kv, pos - s, d, seed=600 + b) * P.BATCH_MAG[b % 3])[0].bfloat16()))
    kc0, vc0 = _padded_cache(krows, T_max), _padded_cache(vrows, T_max)
    ct, st = _tables(nat, d, T_max)
    posd = torch.tensor([pos], dtype=torch.int32, device="cuda")
    ks = torch.tensor(starts, dtype=torch.int32, device="cuda")
    kc1, vc1 = kc0.clone(), vc0.clone()
    q = torch.empty(B, n_h * d, dtype=torch.bfloat16, device="cuda")
    nat.rope_kv_fwd(qkv, q, kc1, vc1, posd, ct, st, qn, kn, eps, 1, n_h, n_kv, d, kv_start=ks)
    for b, s in enumerate(starts):          # the new token alone, plain kernel at position pos - s
        kcx, vcx = torch.zeros(1, n_kv, T_max, d, dtype=torch.bfloat16, device="cuda"), None
        vcx = torch.zeros_like(kcx)
        qx = torch.empty(1, n_h * d, dtype=torch.bfloat16, device="cuda")
        px = torch.tensor([pos - s], dtype=torch.int32, device="cuda")
        nat.rope_kv_fwd(qkv[b:b + 1], qx, kcx, vcx, px, ct, st, qn, kn, eps, 1, n_h, n_kv, d)
        assert torch.equal(_bits(qx), _bits(q[b:b + 1])) and torch.equal(_bits(kcx[0, :, pos - s]), _bits(kc1[b, :, pos]))
    kc2, vc2 = kc0.clone(), vc0.clone()
    out = torch.full((B, n_h * d), NAN, dtype=torch.bfloat16, device="cuda")
    nat.attn_decode_fused(qkv, kc2, vc2, out, posd, ct, st, qn, kn, eps, B, n_h, n_kv, d, scale, kv_start=ks)
    assert torch.equal(_bits(kc1), _bits(kc2)) and torch.equal(_bits(vc1), _bits(vc2))
    for b, s in enumerate(starts):
        qr, kb, vb = q[b:b + 1].view(1, 1, n_h, d), kc1[b:b + 1, :, s:pos + 1], vc1[b:b + 1, :, s:pos + 1]
        ref, _ = ref_fwd(qr, kb, vb, pos - s, scale)
        check_rows(f"{pattern} row {b} start {s}", out[b:b + 1].view(1, 1, n_h, d), ref, oracle_fwd(qr, kb, vb, scale),
                   FWD_K, FWD_FLOOR)
    # all-zero starts: the plain fused kernel's bits
    kc3, vc3, kc4, vc4 = kc1.clone(), vc1.clone(), kc1.clone(), vc1.clone()
    kc3.nan_to_num_(0.0); vc3.nan_to_num_(0.0); kc4.nan_to_num_(0.0); vc4.nan_to_num_(0.0)
    o3, o4 = torch.full_like(out, NAN), torch.full_like(out, NAN)
    nat.attn_decode_fused(qkv, kc3, vc3, o3, posd, ct, st, qn, kn, eps, B, n_h, n_kv, d, scale)
    nat.attn_decode_fused(qkv, kc4, vc4, o4, posd, ct, st, qn, kn, eps, B, n_h, n_kv, d, scale,
                          kv_start=torch.zeros(B, dtype=torch.int32, device="cuda"))
    assert torch.equal(_bits(o3), _bits(o4)) and torch.equal(_bits(kc3), _bits(kc4))
