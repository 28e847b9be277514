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

Also the decode inputs built on these patterns (``decode_inputs``: qkv, q/k-norm gains and a NaN-poisoned cache for
the kernels that rotate q and append the new key themselves) and the forward's row criterion (``check_rows``), shared
by the attention tests on the GPU and the CPU model of the decode chain.
"""
import math

import torch

from oracle import shard_oracle as O

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


# ------------------------------------------------------------------------------------------ decode inputs
def _rms_norm(x, eps):
    return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps)


def decode_inputs(pattern: str, B: int, pos: int, n_h: int, n_kv: int, d: int, qk_norm: bool, T_max: int,
                  eps: float = 1e-6, seed: int = 41):
    """(qkv [B, (n_h+2n_kv)*d], q_norm, k_norm (None without the norm), k_cache, v_cache [B, n_kv, T_max, d]), bf16 on
    the CPU, for one new token per row at `pos`: cached keys 0..pos-1 follow `pattern` over T = pos+1 keys (scaled by
    the query's designed component after the norm), the new key gets its logit through its own designed value, or
    through the k-norm gain when the norm is on; cache rows pos.. are NaN."""
    T = pos + 1
    n_rep, a = n_h // n_kv, designed_dims(d)[0]
    designed = is_designed(pattern)
    z = logit_pattern(pattern, T)
    std = NOISE_STD.get(pattern, NOISE_STD_DESIGNED)
    g = torch.Generator().manual_seed(seed + pos)
    qkv = torch.randn(B, n_h + 2 * n_kv, d, generator=g) * std
    qkv[:, n_h + n_kv:] = make_v(B, n_kv, 1, d, seed=seed + 1 + pos).view(B, n_kv, d).float()
    qn = kn = None
    if qk_norm:
        qn, kn = (1 + 0.1 * torch.randn(d, generator=g)), (1 + 0.1 * torch.randn(d, generator=g))
    if designed:
        qkv[:, :n_h, a] = math.sqrt(d)
        qkv[:, n_h:n_h + n_kv, a] = 1.0
        if qk_norm:
            qn[a] = 1.0
    qkv = qkv.bfloat16()
    # the query's designed component as the kernel will see it (norm; RoPE leaves it within 4e-3 rad)
    qa = qkv[:, :n_h].float()
    if qk_norm:
        qa = _rms_norm(qa, eps) * qn.bfloat16().float()
    qa = qa[..., a].view(B, n_kv, n_rep).mean(-1)                     # [B, n_kv]
    if designed:
        target = z[pos].item() * math.sqrt(d)                         # wanted k_a of the new key times q_a
        if qk_norm:
            kr = _rms_norm(qkv[:, n_h:n_h + n_kv].float(), eps)[..., a].mean().item()
            kn[a] = target / qa.mean().item() / kr
        else:
            qkv[:, n_h:n_h + n_kv, a] = (target / qa).bfloat16()
    qkv = qkv.reshape(B, -1)
    qn = qn.bfloat16() if qk_norm else None
    kn = kn.bfloat16() if qk_norm else None
    kc0 = torch.full((B, n_kv, T_max, d), float("nan"), dtype=torch.bfloat16)
    vc0 = torch.full_like(kc0, float("nan"))
    if pos:
        kc0[:, :, :pos] = torch.randn(B, n_kv, pos, d, generator=g) * std
        if designed:
            kc0[:, :, :pos, a] = (z[:pos].view(1, 1, pos) * math.sqrt(d) / qa.double()[..., None]).bfloat16()
        vc0[:, :, :pos] = make_v(B, n_kv, pos, d, seed=seed + 2 + pos)
    return qkv, qn, kn, kc0, vc0


# ------------------------------------------------------------------------------------------ forward references and criterion
FWD_K, FWD_FLOOR = 2.0, 2e-3     # calibration: tests/test_attention_numerics_gpu.py


def ref_fwd(q, k, v, past, scale):
    """Causal GQA attention in float64: q [B,S,n_h,d], k/v [B,n_kv,T,d] (bf16, on the GPU), queries at positions
    past..past+S-1.  Returns out [B,S,n_h,d] and lse [B,n_h,S] (natural log)."""
    B, S, n_h, d = q.shape
    T, n_rep = k.shape[2], n_h // k.shape[1]
    kk, vv = k.double().repeat_interleave(n_rep, 1), v.double().repeat_interleave(n_rep, 1)
    s = (q.double().transpose(1, 2) @ kk.transpose(2, 3)) * scale
    above = torch.arange(T, device=q.device)[None, :] > torch.arange(past, past + S, device=q.device)[:, None]
    s.masked_fill_(above, float("-inf"))
    lse = torch.logsumexp(s, -1)
    out = torch.exp(s - lse[..., None]) @ vv
    return out.transpose(1, 2), lse


def oracle_fwd(q, k, v, scale):
    """The bf16 yardstick: O.attention_sdpa_math on the CPU (queries are the last S positions of k / v)."""
    n_rep = q.shape[2] // k.shape[1]
    o = O.attention_sdpa_math(q.cpu().transpose(1, 2), k.cpu(), v.cpu(), scale, n_rep)
    return o.view(q.shape)


def row_errors(got, ref, oracle, size=None):
    """Per-row distances to float64 of the kernel and of the oracle; the RMS row norm of the reference and of `size`
    (same shape, or None) within each batch row (the batch rows differ in magnitude on purpose).  Tensors have the
    batch as their first dim."""
    B, d = ref.shape[0], ref.shape[-1]
    rows = lambda x: x.reshape(B, -1, d).to(ref.device, torch.float64)
    rms = lambda x: x.pow(2).sum(-1).mean(-1, keepdim=True).sqrt().expand(B, x.shape[1]).flatten()
    r = rows(ref)
    e_k = (rows(got) - r).norm(dim=-1).flatten()
    e_o = (rows(oracle) - r).norm(dim=-1).flatten()
    return e_k, e_o, rms(r), rms(rows(size)) if size is not None else torch.zeros_like(e_k)


def check_rows(what, got, ref, oracle, k, floor, size=None, cancel=0.0):
    """Each row: |got - ref| <= k |oracle - ref| + floor * RMS(ref) + cancel * RMS(size).  Returns the worst ratio."""
    assert bool(torch.isfinite(got).all()), f"{what}: {int((~torch.isfinite(got)).sum())} non-finite values"
    e_k, e_o, rms, rms_size = row_errors(got, ref, oracle, size)
    bound = k * e_o + floor * rms + cancel * rms_size
    ratio = e_k / bound
    worst = int(ratio.argmax())
    assert float(ratio[worst]) <= 1.0, (f"{what}: row {worst} (of {ratio.numel()}) error {float(e_k[worst]):.3e} > bound "
                                        f"{float(bound[worst]):.3e} ({k} x oracle {float(e_o[worst]):.3e} + floors)")
    return float(ratio[worst])
