"""Score patterns for the attention numerics tests: bf16 q and k whose scaled logits follow a named shape.

Unit-variance q and k give every row a logit spread of about 1, where the online-softmax bookkeeping (running max,
rescale factor, merged split states) hardly matters: a kernel that subtracts the wrong max still returns the right
answer.  The patterns here make that bookkeeping carry the result.

A pattern is a designed logit z(j) per key j (natural-log units, the same for every query) plus random noise on the
other dimensions.  It is written into two head dimensions, `a = d/2 - 1` (coarse) and `b = d - 1` (fine): the lowest-
frequency rotary pair, which RoPE at rope_theta = 1e6 turns by less than 4e-3 rad up to position 2047, so the fused
decode kernel (which rotates q and the new key itself) sees the same shape.  The key side holds small integers, exact in
bf16; the query side holds the scale:  z(j) = (q_a * k_a(j) + q_b * k_b(j)) / sqrt(d).

  flat      today's inputs (unit-variance q and k), the control
  sink      key 0 is L_SINK above the rest for every query
  rising    z(j) = RISE_TILE * (j // 64) + RISE_KEY * (j % 64): every 64-key tile raises each row's running max by more
            than 128 exp2 units (what fp32 can absorb), and under the causal mask each row's own key dominates
  falling   -rising: every tile after the first underflows to zero
  spike@j   one key L_SPIKE above the rest; j may be written T-n (n keys before the end)
  wide      logits with a standard deviation of about 8
"""
import math

import torch

TILE = 64                   # key tile of the prefill kernels and of attn_decode_mma_kernel's ring
WARP_KEYS = 16              # keys of one warp's slice of a tile in attn_decode_mma_kernel
CHUNK_SIMT, CHUNK_MMA = 128, 256      # keys per split of the two decode split kernels
L_SINK, L_SPIKE = 40.0, 100.0         # 100 nats = 144 exp2 units: exp2 of it overflows fp32
RISE_TILE, RISE_KEY = 200.0, 1.0
NOISE_STD = {"flat": 1.0, "wide": 8.0 ** 0.5}      # per-element std of q and k; logits get std NOISE**2
NOISE_STD_DESIGNED = 0.3
BATCH_MAG = (1.0, 8.0, 0.125)         # per batch row factor on V (and dO): leakage across rows shows up per row

PATTERNS = ("flat", "sink", "rising", "falling", "spike", "wide")


def designed_dims(d):
    return d // 2 - 1, d - 1


def spike_pos(pattern: str, T: int) -> int:
    """Key index of a 'spike@j' / 'spike@T-n' pattern over T keys."""
    s = pattern.split("@", 1)[1]
    j = T - int(s[2:]) if s.startswith("T-") else int(s)
    assert 0 <= j < T, (pattern, T)
    return j


def _key_coeffs(pattern: str, T: int):
    """(per-key coarse and fine integers k_a, k_b; logit per unit of each, in nats) of a designed pattern."""
    j = torch.arange(T)
    ka, kb = torch.zeros(T), torch.zeros(T)
    if pattern == "sink":
        ka[0] = 1.0
        return ka, kb, L_SINK, 0.0
    if pattern in ("rising", "falling"):
        sign = 1.0 if pattern == "rising" else -1.0
        return (j // TILE).float(), (j % TILE).float(), sign * RISE_TILE, sign * RISE_KEY
    if pattern.startswith("spike@"):
        ka[spike_pos(pattern, T)] = 1.0
        return ka, kb, L_SPIKE, 0.0
    raise ValueError(pattern)


def is_designed(pattern: str) -> bool:
    return pattern not in NOISE_STD


def logit_pattern(pattern: str, T: int) -> torch.Tensor:
    """The intended designed logit z(j) of keys 0..T-1, float64 (zeros for flat and wide)."""
    if not is_designed(pattern):
        return torch.zeros(T, dtype=torch.float64)
    ka, kb, ca, cb = _key_coeffs(pattern, T)
    return ca * ka.double() + cb * kb.double()


def make_qk(pattern: str, B: int, S: int, T: int, n_h: int, n_kv: int, d: int, seed: int = 0):
    """q [B,S,n_h,d] and k [B,n_kv,T,d] in bf16 (CPU) whose logits q.k / sqrt(d) follow `pattern` plus noise."""
    g = torch.Generator().manual_seed(seed)
    std = NOISE_STD.get(pattern, NOISE_STD_DESIGNED)
    q = torch.randn(B, S, n_h, d, generator=g) * std
    k = torch.randn(B, n_kv, T, d, generator=g) * std
    if is_designed(pattern):
        a, b = designed_dims(d)
        ka, kb, ca, cb = _key_coeffs(pattern, T)
        q[..., a], q[..., b] = ca * math.sqrt(d), cb * math.sqrt(d)
        k[..., a], k[..., b] = ka, kb
    return q.bfloat16(), k.bfloat16()


def make_v(B: int, n_kv: int, T: int, d: int, seed: int = 0) -> torch.Tensor:
    """Unit-variance values, scaled per batch row by BATCH_MAG (powers of two: exact in bf16)."""
    g = torch.Generator().manual_seed(seed + 7919)
    mag = torch.tensor([BATCH_MAG[i % len(BATCH_MAG)] for i in range(B)]).view(B, 1, 1, 1)
    return (torch.randn(B, n_kv, T, d, generator=g) * mag).bfloat16()


def logits(q: torch.Tensor, k: torch.Tensor, past: int) -> torch.Tensor:
    """Scaled float64 logits [B,n_h,S,T] of bf16 q [B,S,n_h,d] over k [B,n_kv,T,d], causal keys only (-inf above)."""
    B, S, n_h, d = q.shape
    T = k.shape[2]
    kk = k.double().repeat_interleave(n_h // k.shape[1], dim=1)
    s = (q.double().transpose(1, 2) @ kk.transpose(2, 3)) * d ** -0.5
    above = torch.arange(T, device=q.device)[None, :] > torch.arange(past, past + S, device=q.device)[:, None]
    return s.masked_fill(above, float("-inf"))
