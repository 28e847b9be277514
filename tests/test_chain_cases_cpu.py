"""The decode chain's launcher arithmetic restated in tests/chain_cases.py: hand-checked geometries, the library's own
answer over a sweep, the attention key partition, and planted faults in the CPU model of the attention job that the
GPU cases' patterns and positions catch.  No GPU."""
import pytest
import torch

from tensorlink_b200.ml import configs as C
from tests import attn_patterns as P
from tests import chain_cases as CC

SMS = 132           # H100 SXM


def _linears(cfg):
    """(name, N, K) of the four decode Linears of a layer"""
    return [("qkv", cfg.qkv_dim, cfg.hidden), ("o", cfg.hidden, cfg.q_dim), ("gu", 2 * cfg.intermediate, cfg.hidden),
            ("down", cfg.hidden, cfg.intermediate)]


def _layer_geometry(cfg, M, stage_kb=0):
    return CC.ring_geometry(M, max(cfg.hidden, cfg.q_dim, cfg.intermediate), stage_kb)


def test_pinned_geometries():
    g = _layer_geometry(C.QWEN25_05B, 1)          # K_max 4864: 9,728 B of x, 218 KB left for 8 slots
    assert g == {"stage_bytes": 24 * 1024, "n_stages": 8, "NW": 8, "kc": 6144}
    assert not any(CC.gemv_units(N, K, g, SMS)["chunked"] for _, N, K in _linears(C.QWEN25_05B))
    g = _layer_geometry(C.QWEN25_7B, 1)           # K_max 18,944: 20 KB slots, the down projection in 4 chunks of 5,120
    assert (g["stage_bytes"], g["n_stages"], g["NW"], g["kc"]) == (20 * 1024, 8, 8, 5120)
    units = {n: CC.gemv_units(N, K, g, SMS) for n, N, K in _linears(C.QWEN25_7B)}
    assert units["down"]["chunked"] and units["down"]["n_chunks"] == 4
    assert not units["qkv"]["chunked"] and units["qkv"]["P"] == 1      # 4 * 3584 B = 14 KB: one pair per 20 KB slot
    g = _layer_geometry(C.QWEN25_7B, 3)           # 113,664 B of x: below 12 KB per slot of 8, so 16 KB slots
    assert (g["stage_bytes"], g["n_stages"], g["NW"]) == (16 * 1024, 5, 5)
    assert _layer_geometry(C.QWEN25_7B, 4) is None    # 175,488 B fixed: 3 slots of 16 KB fit, 4 needed
    assert CC.fixed_bytes(4, 18944) == 175488
    g = _layer_geometry(C.QWEN3_8B, 1)
    assert CC.gemv_units(4096, 12288, g, SMS)["chunked"]


@pytest.mark.parametrize("stage_kb", [0, 3, 8, 9, 11, 12, 16, 20, 24, 40])
def test_model_matches_the_library(stage_kb):
    """the launcher's geometry (tl_decode_chain_geometry, host arithmetic) equals the model everywhere"""
    from tensorlink_b200 import native as nat
    for M in range(1, 5):
        for K in list(range(8, 2048, 8)) + list(range(2048, 32768, 264)) + [4864, 12288, 18944, 18952]:
            g = CC.ring_geometry(M, K, stage_kb)
            lib = nat.decode_chain_geometry(M, K, stage_kb)
            want = None if g is None else (g["stage_bytes"], g["n_stages"], g["NW"], g["kc"])
            assert lib == want, (M, K, stage_kb, lib, want)


def test_forced_slots_reach_every_warp_count():
    """the TL_CHAIN_STAGE_KB values of tests/chain_env_worker.py put NW at 4..8 on the 0.5B layer at M = 1"""
    from tests.chain_env_worker import STAGE_KB
    nws = {CC.ring_geometry(1, 4864, kb)["NW"] for kb in STAGE_KB.values()}
    assert nws == {4, 5, 6, 7, 8}, nws


def test_kc_edges():
    for M in range(1, 5):
        for pairs in (1, 2, 8):
            K = CC.kc_edge(M, pairs=pairs)
            g0, g1 = CC.ring_geometry(M, K), CC.ring_geometry(M, K + 8)
            u0, u1 = CC.gemv_units(64, K, g0, SMS), CC.gemv_units(64, K + 8, g1, SMS)
            if pairs == 1:
                assert not u0["chunked"] and u1["chunked"] and u1["n_chunks"] == 2
                assert 4 * K == g0["stage_bytes"] and K == g0["kc"]
            else:
                assert u0["P"] >= pairs and u1["P"] < pairs


def test_units_partial_and_sparse():
    g = CC.ring_geometry(1, 24)
    u = CC.gemv_units(2 * (8 * 5 + 3), 24, g, SMS)
    assert u["P"] == 8 and u["units"] == 6 and u["last_unit_pairs"] == 3
    u = CC.gemv_units(10, 8, CC.ring_geometry(2, 8), SMS)
    assert u["units"] == 1 and sum(b - a for a, b in u["u_ranges"]) == 1


def test_attention_partition_pinned():
    p = CC.attn_partition(SMS, 2, 1, 127)
    assert (p["cpg"], p["cpg_eff"], p["chunk"], p["ranges"], p["combine"]) == (66, 1, 128, [(0, 128)], False)
    p = CC.attn_partition(SMS, 2, 1, 128)
    assert (p["cpg_eff"], p["chunk"], p["ranges"], p["owner"]) == (2, 96, [(0, 96), (96, 129)], 1)
    p = CC.attn_partition(SMS, 2, 1, 8191)
    assert (p["cpg_eff"], p["chunk"]) == (64, 128)
    p = CC.attn_partition(SMS, 4, 3, 8191)                  # 12 groups of 11 CTAs
    assert (p["cpg"], p["cpg_eff"], p["chunk"], p["ranges"][-1]) == (11, 11, 768, (7680, 8192))


@pytest.mark.parametrize("sms", [132, 114, 78])
def test_attention_partition_covers_every_key_once(sms):
    g = torch.Generator().manual_seed(sms)
    for _ in range(300):
        n_kv = int(torch.randint(1, 9, (1,), generator=g))
        M = int(torch.randint(1, 5, (1,), generator=g))
        pos = int(torch.randint(0, 20000, (1,), generator=g))
        p = CC.attn_partition(sms, n_kv, M, pos)
        r = p["ranges"]
        assert r[0][0] == 0 and r[-1][1] == pos + 1 and len(r) == p["cpg_eff"] <= p["cpg"]
        assert all(a < b for a, b in r) and all(r[i][1] == r[i + 1][0] for i in range(len(r) - 1))
        assert all(a % CC.DC_TILE == 0 for a, _ in r)
        assert p["cpg_eff"] <= -(-(pos + 1) // CC.DC_MIN_KEYS)        # a CTA per 128 keys at most


# ------------------------------------------------------------------------------------------------ planted faults
def _model_case(n_h, n_kv, d, M, pos, pattern, fault):
    """row 0 through the CPU model, against float64 and the bf16 oracle.  q and the new key are taken as already
    rotated (the model has no RoPE), so the case runs without the q/k-norm."""
    qkv, _, _, kc, vc = P.decode_inputs(pattern, 1, pos, n_h, n_kv, d, False, pos + 1)
    x = qkv.view(n_h + 2 * n_kv, d)
    q, k_new, v_new = x[:n_h], x[n_h:n_h + n_kv], x[n_h + n_kv:]
    kc, vc = kc.clone(), vc.clone()
    scale, n_rep = d ** -0.5, n_h // n_kv
    part = CC.attn_partition(SMS, n_kv, M, pos)
    out = torch.stack([CC.chain_attention(q[h * n_rep:(h + 1) * n_rep], kc[0, h], vc[0, h], k_new[h], v_new[h], pos,
                                          scale, part, fault) for h in range(n_kv)]).view(1, 1, n_h, d)
    kc[0, :, pos], vc[0, :, pos] = k_new, v_new
    qr, k, v = q.view(1, 1, n_h, d), kc[:, :, :pos + 1], vc[:, :, :pos + 1]
    ref, _ = P.ref_fwd(qr, k, v, pos, scale)
    try:
        P.check_rows(pattern, out, ref, P.oracle_fwd(qr, k, v, scale), P.FWD_K, P.FWD_FLOOR)
        return True
    except AssertionError:
        return False


def _fault_cases():
    """the GPU cases the CPU model can afford (contexts up to 1,024 keys), by geometry with the norm off"""
    return [c for c in CC.attn_cases(SMS) if c[5] <= 1024]


def test_unfaulted_model_meets_the_criterion():
    bad = [c for c in _fault_cases() if not _model_case(c[0], c[1], c[2], c[4], c[5], c[6], None)]
    assert not bad, bad[:5]


@pytest.mark.parametrize("fault", CC.FAULTS)
def test_planted_fault_is_caught(fault):
    caught = [c for c in _fault_cases() if not _model_case(c[0], c[1], c[2], c[4], c[5], c[6], fault)]
    assert caught, f"no case of attn_cases catches {fault}"
    print(fault, "caught by", len(caught), "cases, e.g.", caught[:3])
