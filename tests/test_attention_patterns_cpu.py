"""The score patterns of tests/attn_patterns.py have the property each is named for, and they expose a fault in the
online-softmax bookkeeping that unit-variance inputs hide (a tiled CPU model with a stale running max).  No GPU."""
import pytest
import torch

from oracle import shard_oracle as O
from tests import attn_patterns as P

LOG2E = 1.4426950408889634
FP32_EXP2_RANGE = 128.0          # exp2 of more than this overflows fp32


def _case(pattern, B=1, S=130, past=60, n_h=2, n_kv=1, d=64, seed=3):
    q, k = P.make_qk(pattern, B, S, past + S, n_h, n_kv, d, seed=seed)
    return q, k, P.logits(q, k, past)


@pytest.mark.parametrize("d", [64, 128])
def test_flat_and_wide_spread(d):
    for pattern, want in (("flat", 1.0), ("wide", 8.0)):
        _, _, s = _case(pattern, d=d, past=0, S=256)
        sd = s[torch.isfinite(s)].std().item()
        assert 0.85 * want < sd < 1.15 * want, (pattern, sd)


@pytest.mark.parametrize("d,past", [(64, 0), (128, 37), (128, 300)])
def test_rising_raises_every_tiles_max_past_fp32_range(d, past):
    S = 200
    _, _, s = _case("rising", S=S, past=past, d=d)
    T = past + S
    s2 = s * LOG2E                                               # the kernels' log2 domain
    for t in range(1, (T + P.TILE - 1) // P.TILE):
        prev = s2[..., : t * P.TILE].amax(-1)                     # running max after tile t-1
        tile = s2[..., t * P.TILE:(t + 1) * P.TILE]
        sees = torch.isfinite(tile[..., 0])                       # rows whose causal limit reaches tile t
        rise = tile.amax(-1) - prev
        assert bool(sees.any()) and bool((rise[sees] > 1.4 * FP32_EXP2_RANGE).all()), (t, rise[sees].min())
    # under the causal mask each row's own key dominates
    assert torch.equal(s.argmax(-1)[0, 0], torch.arange(past, T))
    mass = torch.softmax(s, -1).diagonal(offset=past, dim1=-2, dim2=-1)
    assert bool((mass > 0.5).all())


def test_falling_underflows_every_later_tile():
    _, _, s = _case("falling", S=300, past=0, d=128)
    p = torch.exp((s - s.amax(-1, keepdim=True)).float())         # fp32, as the kernels exponentiate
    assert bool((p[..., P.TILE:] == 0).all())
    assert bool((s.argmax(-1) == 0).all())


@pytest.mark.parametrize("S,past", [(300, 0), (1, 4095)])
def test_sink_holds_the_mass_on_key0(S, past):
    _, _, s = _case("sink", S=S, past=past, d=128)
    assert bool((torch.softmax(s, -1)[..., 0] >= 0.99).all())


# spike position -> (64-key tile, warp slice of attn_decode_mma_kernel, split of the simt kernel, split of the mma kernel)
SPIKES = {"spike@63": (0, 3, 0, 0), "spike@64": (1, 0, 0, 0), "spike@65": (1, 0, 0, 0), "spike@127": (1, 3, 0, 0),
          "spike@128": (2, 0, 1, 0), "spike@129": (2, 0, 1, 0), "spike@255": (3, 3, 1, 0), "spike@256": (4, 0, 2, 1),
          "spike@257": (4, 0, 2, 1), "spike@50": (0, 3, 0, 0), "spike@305": (4, 3, 2, 1)}


@pytest.mark.parametrize("pattern", sorted(SPIKES))
def test_spike_lands_where_the_kernels_split_work(pattern):
    T = 320
    j = P.spike_pos(pattern, T)
    assert (j // P.TILE, j % P.TILE // P.WARP_KEYS, j // P.CHUNK_SIMT, j // P.CHUNK_MMA) == SPIKES[pattern]
    _, _, s = _case(pattern, S=1, past=T - 1, d=128)
    top2 = s.topk(2, -1)
    assert bool((top2.indices[..., 0] == j).all())
    assert bool((top2.values[..., 0] - top2.values[..., 1] > P.L_SPIKE - 2).all())
    assert P.spike_pos("spike@T-1", T) == T - 1 and P.spike_pos("spike@T-2", T) == T - 2


def test_patterns_are_exact_in_bf16():
    """The designed key coordinates are small integers (exact in bf16), so the logits follow z(j) to the rounding of
    the query scale and the noise."""
    for pattern in ("sink", "rising", "falling", "spike@65"):
        T = 600
        q, k = P.make_qk(pattern, 1, 1, T, 1, 1, 128, seed=5)
        a, b = P.designed_dims(128)
        z = (q[0, 0, 0, a].double() * k[0, 0, :, a].double() + q[0, 0, 0, b].double() * k[0, 0, :, b].double()) / 128 ** 0.5
        want = P.logit_pattern(pattern, T)
        assert torch.allclose(z, want, rtol=4e-3, atol=0), pattern


def test_batch_rows_differ_in_magnitude():
    v = P.make_v(3, 2, 50, 64)
    rms = v.float().pow(2).mean((1, 2, 3)).sqrt()
    assert torch.allclose(rms, torch.tensor(P.BATCH_MAG), rtol=0.1)


# ------------------------------------------------------------------------------------------ stale-max guard
def online_softmax(q, k, v, past, stale):
    """Tiled online softmax in the kernels' numerics (64-key tiles, log2 domain, P rounded to bf16 for P.V).  With
    stale=True it keeps subtracting the first max it saw and never rescales (alpha = 1): exact for any fixed max,
    short of overflow."""
    B, S, n_h, d = q.shape
    T = past + S
    n_rep = n_h // k.shape[1]
    vv = O.repeat_kv(v, n_rep).float()
    s = P.logits(q, k, past).float() * LOG2E
    m = torch.full(s.shape[:-1], float("-inf"))
    l, o = torch.zeros(s.shape[:-1]), torch.zeros(*s.shape[:-1], d)
    for t0 in range(0, T, P.TILE):
        st = s[..., t0:t0 + P.TILE]
        m_new = torch.maximum(m, st.amax(-1))
        if stale:
            m_new = torch.where(m == float("-inf"), m_new, m)
        msub = torch.where(m_new == float("-inf"), 0.0, m_new)
        alpha = torch.exp2(m - msub)
        p = torch.exp2(st - msub[..., None])
        l = l * alpha + p.sum(-1)
        o = o * alpha[..., None] + p.bfloat16().float() @ vv[..., t0:t0 + P.TILE, :]
        m = m_new
    return (o / l[..., None]).transpose(1, 2).reshape(B, S, -1)


@pytest.mark.parametrize("B,S,past,n_h,n_kv,d", [(2, 257, 0, 8, 2, 128), (1, 130, 300, 7, 1, 128)])
def test_stale_max_model_hides_on_flat_and_overflows_on_rising(B, S, past, n_h, n_kv, d):
    v = P.make_v(B, n_kv, past + S, d, seed=1)
    for pattern in ("flat", "rising"):
        q, k = P.make_qk(pattern, B, S, past + S, n_h, n_kv, d, seed=2)
        exact = torch.softmax(P.logits(q, k, past), -1) @ O.repeat_kv(v, n_h // n_kv).double()
        exact = exact.transpose(1, 2).reshape(B, S, -1)
        good = online_softmax(q, k, v, past, stale=False)
        assert O.rel_l2(good, exact) < 4e-3, pattern                    # the model itself is right
        bad = online_softmax(q, k, v, past, stale=True)
        if pattern == "flat":
            assert bool(torch.isfinite(bad).all()) and O.rel_l2(bad, exact) < 4e-3
        else:
            assert not bool(torch.isfinite(bad).all())
