"""``tl_attn_bwd_rows`` (the attention backward of a left-padded training batch) row by row against float64, on the
peaked score patterns of tests/attn_patterns.py, into gradient buffers that start as NaN.

tests/test_attention_bwd_rows_gpu.py holds the padded backward to one rel-L2 bound over all real rows of random,
std-0.7 inputs: on flat scores a wrong running max or lse cancels out, and one bad row (the first real query row of a
tile, say) is lost in a whole-tensor norm.  Here every batch row b gets its own start s_b, and its real part (positions
[s_b, S)) is built as a sequence of its own: q and k from ``P.make_qk(pattern, 1, L_b, L_b, ...)``, so 'sink' is the
row's first real key (mid-tile for most starts); v and dO from ``P.make_v`` times ``P.BATCH_MAG[b]``, so a read across
batch rows shows up in the row read into.  Spikes sit at absolute tile edges: spike@63 / spike@64 on the first key at or
after s_b that lies 63 / 64 modulo 64 (the last key when none does), spike@T-1 on key S-1.  Pad q, dO, out and lse rows
and the K/V slots below s_b are NaN, which the header allows.  The forward is the kernel's own (``attn_prefill_fwd``
with ``kv_start``), as in training, and the backward consumes its out and lse.

Starts are distinct within a batch: 0, 1, 63, 64, 65, 127, 128, 129 and S-1 (one real token), those below S, at
S in {64, 65, 128, 130, 200, 257}: the tile edges where the kernels' first key tile (k_start / 64), the partial first
key tile and the partial last query tile meet.

Criteria, per batch row, under TL_ATTN_BWD = TL_ATTN_IMPL = mma and = wgmma:
  * dq, dk and dv start as NaN, as training's torch.empty buffers may: dq is exactly 0 on pad query rows, every
    per-head dk / dv partial is exactly 0 on slots below s_b, and every slot of [0, S) is finite, so every one of them
    was written;
  * real rows of dq, dk and dv (dk / dv summed over the GQA group) meet the bound of
    tests/test_attention_numerics_gpu.py (BWD_K, BWD_FLOOR, BWD_CANCEL) against float64 ``ref_bwd`` of the row's real
    part alone: the unpadded causal backward of [s_b, S) at past 0;
  * slots [S, T_max) of dk / dv keep what the caller left there (T_max = S + 64 in ``test_bwd_rows_past_s``);
  * the start-0 row equals ``tl_attn_bwd`` on that row alone (same q, K/V, out, dO, lse) bit for bit.  No reduction
    depends on B: every CTA owns one (tile, query head, batch row), the D = rowsum(dO * O) pass is one warp per
    (row, position, head), and the query rows past S that the last tile's TMA box reaches (the next batch row's, or
    out of bounds) meet only zero P and dS, and are zeroed first in the left-padded dK/dV kernel.

Measured on an H100 80GB HBM3 (700 W power limit); worst error / bound over the file, per backward form:
  mma    dq 0.63, dk 0.39, dv 0.24
  wgmma  dq 0.63, dk 0.39, dv 0.24   (the S = 4096 case alone: dq 0.52, dk 0.31, dv 0.23)
The two forms give the same worst rows: dq on 'rising' at S = 257, dk on 'rising' and dv on 'wide' at S = 65.  The
bounds are the numerics file's, not re-tuned.  The file runs in about 20 s there (101 tests).
"""
import pytest
import torch

from tests import attn_patterns as P
from tests.test_attention_numerics_gpu import BWD_CANCEL, BWD_FLOOR, BWD_K, NAN, check_rows, oracle_bwd, ref_bwd

pytestmark = pytest.mark.gpu

IMPLS = ["mma", "wgmma"]
GEOMS = [(14, 2, 64), (28, 4, 128), (32, 8, 128), (4, 4, 64), (7, 1, 128)]      # n_rep 7, 7, 4, 1, 7 on one KV head
SEQS = [64, 65, 128, 130, 200, 257]
PATTERNS = ["flat", "sink", "rising", "falling", "spike@63", "spike@64", "spike@T-1", "wide"]
# every pattern at every S, the geometry turning with both: each pattern meets every geometry, and so does each S
CASES = [(*GEOMS[(i + j) % len(GEOMS)], S, pat) for i, pat in enumerate(PATTERNS) for j, S in enumerate(SEQS)]


@pytest.fixture(scope="module")
def nat():
    from tensorlink_b200 import native
    native.require_device()
    return native


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def starts_for(S):
    """Distinct starts at the tile edges, and S - 1 (one real token); all below S."""
    out = []
    for s in (0, 1, 63, 64, 65, 127, 128, 129, S - 1):
        if s < S and s not in out:
            out.append(s)
    return out


def row_pattern(pattern, S, s):
    """The pattern of a row's real keys [s, S), relative to its first real key: spike@63 / spike@64 move to the first
    absolute position at or after s that lies 63 / 64 modulo the tile (S - 1 when none is below S)."""
    if not pattern.startswith("spike@") or pattern.endswith("T-1"):
        return pattern
    j = int(pattern.split("@")[1])
    p = j if s <= j else s + (j - s) % P.TILE
    return f"spike@{min(p, S - 1) - s}"


def _first(mask):
    """index tuple of the first True of a bool tensor"""
    return tuple(int(i) for i in mask.nonzero()[0])


def _case(nat, impl, n_h, n_kv, d, S, pattern, starts, T_max=None):
    """One left-padded batch, forward then backward; every criterion of the module docstring.  Returns the worst
    error / bound of dq, dk and dv over the batch rows."""
    T_max = T_max or S                                    # training's layout: dk / dv hold exactly S slots
    B, scale, n_rep = len(starts), d ** -0.5, n_h // n_kv
    q = torch.full((B, S, n_h, d), NAN, dtype=torch.bfloat16)
    do = torch.full_like(q, NAN)
    kc = torch.full((B, n_kv, T_max, d), NAN, dtype=torch.bfloat16)
    vc = torch.full_like(kc, NAN)
    for b, s in enumerate(starts):
        L, mag = S - s, P.BATCH_MAG[b % len(P.BATCH_MAG)]
        qb, kb = P.make_qk(row_pattern(pattern, S, s), 1, L, L, n_h, n_kv, d, seed=50 + b)
        q[b, s:], kc[b, :, s:S] = qb[0], kb[0]
        vc[b, :, s:S] = P.make_v(1, n_kv, L, d, seed=60 + b)[0] * mag
        do[b, s:] = P.make_v(1, L, n_h, d, seed=70 + b)[0] * mag
    q, do, kc, vc = q.cuda(), do.cuda(), kc.cuda(), vc.cuda()
    ks = torch.tensor(starts, dtype=torch.int32, device="cuda")
    pad = (torch.arange(S)[None, :] < torch.tensor(starts)[:, None]).cuda()          # [B, S] pad query rows

    out = torch.full((B, S, n_h * d), NAN, dtype=torch.bfloat16, device="cuda")
    lse = torch.full((B, n_h, S), NAN, dtype=torch.float32, device="cuda")
    nat.attn_prefill_fwd(q, kc, vc, out, lse, B, S, 0, n_h, n_kv, d, scale, kv_start=ks)
    out[pad] = NAN                                        # pad rows of out and lse may hold anything
    lse.transpose(1, 2)[pad] = NAN
    dq = torch.full((B, S, n_h, d), NAN, dtype=torch.bfloat16, device="cuda")
    dk = torch.full((B, n_h, T_max, d), NAN, dtype=torch.bfloat16, device="cuda")      # one partial per query head
    dv = torch.full_like(dk, NAN)
    ws = torch.empty(nat.attn_bwd_ws(B, S, n_h), dtype=torch.uint8, device="cuda")
    nat.attn_bwd(q, kc, vc, out, do.view(B, S, n_h * d), lse, dq, dk, dv, ws, B, S, n_h, n_kv, d, scale, kv_start=ks)

    tag = f"{impl} {pattern} S={S} n_h={n_h} n_kv={n_kv} d={d}"
    for name, g in (("dk", dk), ("dv", dv)):
        bad = ~torch.isfinite(g[:, :, :S])
        if bool(bad.any()):
            b, h, t = _first(bad)[:3]
            raise AssertionError(f"{tag} row {b} start {starts[b]}: {name} head {h} slot {t} not finite "
                                 f"({int(bad.any(-1).sum())} slots), not written")
        assert torch.equal(_bits(g[:, :, S:]), _bits(torch.full_like(g[:, :, S:], NAN))), \
            f"{tag}: {name} slots past S = {S} written"
    dks = dk.float().view(B, n_kv, n_rep, T_max, d).sum(2)
    dvs = dv.float().view(B, n_kv, n_rep, T_max, d).sum(2)
    worst = {"dq": 0.0, "dk": 0.0, "dv": 0.0}
    for b, s in enumerate(starts):
        what = f"{tag} row {b} start {s}"
        if s:
            nz = dq[b, :s] != 0
            assert not bool(nz.any()), f"{what}: dq pad query row {_first(nz)[0]} not zero"
            for name, g in (("dk", dk), ("dv", dv)):
                nz = g[b, :, :s] != 0
                assert not bool(nz.any()), f"{what}: {name} head {_first(nz)[0]} pad slot {_first(nz)[1]} not zero"
        real = (q[b:b + 1, s:], kc[b:b + 1, :, s:S], vc[b:b + 1, :, s:S], do[b:b + 1, s:], scale)
        refs, sizes = ref_bwd(*real)
        gots = (dq[b:b + 1, s:], dks[b:b + 1, :, s:S], dvs[b:b + 1, :, s:S])
        for name, got, ref, oracle, size in zip(("dq", "dk", "dv"), gots, refs, oracle_bwd(*real), sizes):
            r = check_rows(f"{what} {name}", got, ref, oracle, BWD_K, BWD_FLOOR, size, BWD_CANCEL)
            worst[name] = max(worst[name], r)

    b0 = starts.index(0)                                  # the start-0 row against the plain backward on it alone
    one = lambda t: t[b0:b0 + 1].contiguous()
    dq1, dk1, dv1 = torch.full_like(one(dq), NAN), torch.full_like(one(dk), NAN), torch.full_like(one(dv), NAN)
    ws1 = torch.empty(nat.attn_bwd_ws(1, S, n_h), dtype=torch.uint8, device="cuda")
    nat.attn_bwd(one(q), one(kc), one(vc), one(out), one(do).view(1, S, n_h * d), one(lse), dq1, dk1, dv1, ws1,
                 1, S, n_h, n_kv, d, scale)
    for name, a, c in (("dq", dq[b0], dq1[0]), ("dk", dk[b0], dk1[0]), ("dv", dv[b0], dv1[0])):
        assert torch.equal(_bits(a), _bits(c)), f"{tag} row {b0} start 0: {name} differs from tl_attn_bwd on the row alone"
    return worst


def _env(monkeypatch, impl):
    monkeypatch.setenv("TL_ATTN_IMPL", impl)
    monkeypatch.setenv("TL_ATTN_BWD", impl)


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("n_h,n_kv,d,S,pattern", CASES)
def test_bwd_rows(nat, monkeypatch, impl, n_h, n_kv, d, S, pattern):
    _env(monkeypatch, impl)
    _case(nat, impl, n_h, n_kv, d, S, pattern, starts_for(S))


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("n_h,n_kv,d,S,pattern", [(14, 2, 64, 130, "spike@64"), (28, 4, 128, 200, "rising")])
def test_bwd_rows_past_s(nat, monkeypatch, impl, n_h, n_kv, d, S, pattern):
    """T_max = S + 64: the K/V slots [S, T_max) are NaN, and the dk / dv slots there keep their NaN."""
    _env(monkeypatch, impl)
    _case(nat, impl, n_h, n_kv, d, S, pattern, starts_for(S), T_max=S + P.TILE)


def test_bwd_rows_long_wgmma(nat, monkeypatch):
    """4096 rising keys: the two-slot TMA ring runs through up to 64 query or key tiles, from a first tile mid-row."""
    _env(monkeypatch, "wgmma")
    _case(nat, "wgmma", 2, 1, 128, 4096, "rising", [0, 1000, 4031])
