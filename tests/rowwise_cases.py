"""Element-by-element checks of the row-wise and element-wise kernels: SwiGLU, RMSNorm, the rotary tables, RoPE + KV
append and its backward, cross-entropy's dlogits, the embedding gather, the gradient commits, the AdamW step and the two
samplers (draw by draw).

Every ``run_*`` function builds one case's inputs, calls the kernel through ``launch`` (``tensorlink_b200.native`` on the
GPU, ``CpuKernels`` here) and compares each output element with a float64 reference under one of three checkers:

  * exact:  the output must equal the reference bit for bit (the reference applies the kernel's rounding points, which
            are HF's);
  * band:   exact, except where the float64 value lies within a stated distance of a bf16 rounding tie; there the other
            neighbour is allowed too (a "flip", counted and reported);
  * guard:  every output lives inside a larger allocation whose pads hold a sentinel pattern, every input inside NaN
            pads; afterwards the pads and the inputs must be unchanged.  Guard pads stay inside one allocation.

Each case states its bound next to the reason for it.  Nothing here needs a GPU: tests/test_rowwise_cases_cpu.py runs
the checkers on ``CpuKernels`` and shows that each planted fault is caught.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

BF16_SENTINEL = 0x7FA5          # a NaN payload no kernel produces
F32_SENTINEL = 0x7FBADBAD
PAD = 64                        # guard elements on each side (keeps 16-byte alignment for bf16 and fp32)
BF16_MAX_NEXT = 2.0 ** 128      # RNE to bf16 overflows to inf from here
FLT_MAX = float(np.finfo(np.float32).max)
_INT = {torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.int64: torch.int64, torch.int32: torch.int32}


# ------------------------------------------------------------------------------------------------ bf16 arithmetic
def _grid(x):
    """(q, step): x / step with step the bf16 spacing at x (subnormals included)"""
    _, e = torch.frexp(x)
    step = torch.ldexp(torch.ones_like(x), (e.to(torch.int64) - 8).clamp_min(-133))
    return x / step, step


def rbf(x) -> torch.Tensor:
    """float64 -> the float64 value of its round-to-nearest-even bf16 (a single rounding, overflow to inf)"""
    x = torch.as_tensor(x, dtype=torch.float64)
    q, step = _grid(x)
    r = torch.round(q) * step                      # torch.round: half to even
    r = torch.where(r.abs() >= BF16_MAX_NEXT, torch.copysign(torch.full_like(r, math.inf), x), r)
    return torch.where(torch.isfinite(x), r, x)


def f32(x) -> torch.Tensor:
    """float64 -> the float64 value of its nearest fp32"""
    return torch.as_tensor(x, dtype=torch.float64).float().double()


def bits(t: torch.Tensor) -> torch.Tensor:
    """bf16 bit patterns (int16) of a bf16 tensor, or of a float64 tensor on the bf16 grid"""
    if t.dtype == torch.float64:
        t = t.to(torch.bfloat16)
    return t.contiguous().view(torch.int16)


def ulp_bf16(x) -> torch.Tensor:
    x = torch.as_tensor(x, dtype=torch.float64).abs()
    _, e = torch.frexp(x)
    return torch.ldexp(torch.ones_like(x), (e.to(torch.int64) - 8).clamp_min(-133))


def ulp_f32(x) -> torch.Tensor:
    x = torch.as_tensor(x, dtype=torch.float64).abs()
    _, e = torch.frexp(x)
    return torch.ldexp(torch.ones_like(x), (e.to(torch.int64) - 24).clamp_min(-149))


def neighbours(x):
    """(nearest bf16, the other bf16 neighbour, |x - the tie between them|)"""
    x = torch.as_tensor(x, dtype=torch.float64)
    q, step = _grid(x)
    lo, hi = torch.floor(q) * step, torch.ceil(q) * step
    near = rbf(x)
    other = torch.where(near == lo, hi, lo)
    tie_dist = (x - (torch.floor(q) + 0.5) * step).abs()
    return near, other, tie_dist


# ------------------------------------------------------------------------------------------------ checkers
def check_exact(name, got, want, errors, limit=5):
    """bit for bit; ``want`` is bf16 or float64 on the bf16 grid"""
    g, w = bits(got.cpu()).reshape(-1), bits(want.cpu()).reshape(-1)
    bad = (g != w).nonzero()[:, 0]
    if len(bad):
        gv, wv = got.cpu().reshape(-1).double(), want.cpu().reshape(-1).double()
        ex = [(int(i), float(gv[i]), float(wv[i])) for i in bad[:limit]]
        errors.append(f"{name}: {len(bad)} of {g.numel()} differ from the exact reference, e.g. (index, got, want) {ex}")
    return int(len(bad))


def check_band(name, got, ref64, width, errors, limit=5):
    """exact outside the band; where |ref64 - tie| <= width the other bf16 neighbour is allowed.  Returns the flip count."""
    ref64 = ref64.reshape(-1)
    near, other, tie = neighbours(ref64)
    width = torch.as_tensor(width, dtype=torch.float64)
    width = width.reshape(-1) if width.numel() == ref64.numel() else width.expand_as(ref64)
    g = bits(got.cpu()).reshape(-1)
    eq, alt = g == bits(near), (g == bits(other)) & (tie <= width)
    bad = (~(eq | alt)).nonzero()[:, 0]
    if len(bad):
        gv = got.cpu().reshape(-1).double()
        ex = [(int(i), float(gv[i]), float(ref64[i]), float(tie[i] / width[i]) if width[i] > 0 else math.inf)
              for i in bad[:limit]]
        errors.append(f"{name}: {len(bad)} of {g.numel()} outside the tie band, e.g. (index, got, float64, tie distance / band) {ex}")
    return int((alt & ~eq).sum())


def check_candidates(name, got, cands, errors, limit=5):
    """each element must equal one of the candidate bf16 values (float64 tensors on the bf16 grid)"""
    g = bits(got.cpu()).reshape(-1)
    ok = torch.zeros_like(g, dtype=torch.bool)
    for c in cands:
        ok |= g == bits(c.reshape(-1))
    bad = (~ok).nonzero()[:, 0]
    if len(bad):
        gv = got.cpu().reshape(-1).double()
        ex = [(int(i), float(gv[i]), float(cands[0].reshape(-1)[i])) for i in bad[:limit]]
        errors.append(f"{name}: {len(bad)} of {g.numel()} match no allowed value, e.g. (index, got, first allowed) {ex}")
    flips = int(((~(g == bits(cands[0].reshape(-1)))) & ok).sum())
    return flips


def check_bound(name, got, ref64, bound, errors, limit=5):
    """|got - ref64| <= bound per element (non-finite output fails); returns max |err| / bound"""
    gv = got.cpu().reshape(-1).double()
    ref64, bound = ref64.reshape(-1), torch.as_tensor(bound, dtype=torch.float64)
    bound = bound.reshape(-1) if bound.numel() == gv.numel() else bound.expand(gv.shape)
    err = (gv - ref64).abs()
    bad = (~(err <= bound)).nonzero()[:, 0]
    if len(bad):
        ex = [(int(i), float(gv[i]), float(ref64[i]), float(bound[i])) for i in bad[:limit]]
        errors.append(f"{name}: {len(bad)} of {gv.numel()} beyond the bound, e.g. (index, got, float64, bound) {ex}")
    r = err / bound
    r = r[torch.isfinite(r)]
    return float(r.max()) if r.numel() else 0.0


class Buf:
    """n elements (``t``) inside one allocation with PAD guard elements on each side, all of it filled with fill_bits
    first; ``pads_changed`` counts guard elements that no longer hold it."""

    def __init__(self, n, dtype, device, fill_bits):
        self.n, self.dtype, self.fill_bits = n, dtype, fill_bits
        self.buf = torch.empty(n + 2 * PAD, dtype=dtype, device=device)
        self.raw = self.buf.view(_INT[dtype])
        self.raw.fill_(fill_bits)
        self.t = self.buf[PAD:PAD + n]

    def pads_changed(self):
        r = self.raw.cpu()
        return int((r[:PAD] != self.fill_bits).sum() + (r[PAD + self.n:] != self.fill_bits).sum())


def nan_bits(dtype):
    return {torch.bfloat16: 0x7FC0, torch.float32: 0x7FC00000}[dtype]


def sentinel_bits(dtype):
    return {torch.bfloat16: BF16_SENTINEL, torch.float32: F32_SENTINEL}[dtype]


def inp(values: torch.Tensor, device) -> Buf:
    """an input copied into a NaN-padded allocation (ids: pads of -1)"""
    dt = values.dtype
    b = Buf(values.numel(), dt, device, -1 if dt in (torch.int64, torch.int32) else nan_bits(dt))
    b.t.copy_(values.reshape(-1).to(device))
    return b


def out(n, dtype, device) -> Buf:
    return Buf(n, dtype, device, sentinel_bits(dtype))


class Guards:
    """the inputs (must be unchanged everywhere) and outputs (pads must keep their sentinel) of one call"""

    def __init__(self):
        self.ins, self.outs = [], []

    def i(self, name, values, device):
        b = inp(values, device)
        self.ins.append((name, b, b.raw.clone()))
        return b

    def o(self, name, n, dtype, device, init: Optional[torch.Tensor] = None):
        b = out(n, dtype, device)
        if init is not None:
            b.t.copy_(init.reshape(-1).to(device))
        self.outs.append((name, b))
        return b

    def check(self, errors, prefix):
        for name, b, snap in self.ins:
            if not torch.equal(b.raw, snap):
                errors.append(f"{prefix}: input {name} was written ({int((b.raw != snap).sum())} elements)")
        for name, b in self.outs:
            n = b.pads_changed()
            if n:
                errors.append(f"{prefix}: {n} guard elements around {name} were written")


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def randn_bf16(shape, seed, scale=1.0):
    return (torch.randn(shape, generator=_gen(seed), dtype=torch.float64) * scale).to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------ SwiGLU
SILU_TIE_REL = 2.0 ** -20       # torch's fp32 silu and the kernel's agree to a few fp32 ulp (2^-21 and below), so their
                                # bf16 roundings may differ only where silu lies this close (relative) to a tie


def finite_bf16_patterns() -> torch.Tensor:
    """every bf16 bit pattern except NaN and +-inf, as a bf16 tensor (65,280 values)"""
    b = torch.arange(65536, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)
    return b[torch.isfinite(b.float())]


def silu64(g64):
    """float64 silu with torch's fp32 overflow: exp(-g) beyond FLT_MAX is inf, so silu(g <= -88.73) is -0"""
    e = torch.exp(-g64)
    e = torch.where(e > FLT_MAX, torch.full_like(e, math.inf), e)
    return g64 / (1.0 + e), 1.0 / (1.0 + e)


@dataclass(frozen=True)
class SwiCase:
    name: str
    M: int
    I: int
    ups: tuple = (1.0, -1.5, 0.3125, 96.0)


def swiglu_cases():
    # M·I/4 vectors: the kernel grid is min(ceil(n_vec/256), 16·SMs) CTAs of 256 threads, so 4864 x 500 runs the
    # grid-stride loop more than once with a ragged last pass; the others end inside the first pass
    return [SwiCase("I4", 65281, 4), SwiCase("I64", 4083, 64), SwiCase("I4864", 500, 4864), SwiCase("I18944", 15, 18944),
            SwiCase("ranges", 7, 4864, ups=())]


def swiglu_inputs(c: SwiCase, seed=11):
    n = c.M * c.I
    if c.ups:   # every finite gate pattern once per up value, then random gates
        pats = finite_bf16_patterns()
        g = torch.cat([pats] * len(c.ups))
        u = torch.cat([torch.full((pats.numel(),), v, dtype=torch.bfloat16) for v in c.ups])
        if g.numel() < n:
            rest = n - g.numel()
            g = torch.cat([g, randn_bf16(rest, seed, 4.0)])
            u = torch.cat([u, randn_bf16(rest, seed + 1)])
        g, u = g[:n], u[:n]
    else:       # distinct ranges: gates in [-6, -1], ups in [16, 64); a swap of the two cannot pass
        r = torch.rand(n, generator=_gen(seed), dtype=torch.float64)
        g = (-1.0 - 5.0 * r).to(torch.bfloat16)
        u = (16.0 * 4.0 ** torch.rand(n, generator=_gen(seed + 1), dtype=torch.float64)).to(torch.bfloat16)
    gu = torch.stack([g, u], 1).reshape(c.M, 2 * c.I)
    dh = randn_bf16((c.M, c.I), seed + 2, 2.0)
    return gu, dh


def run_swiglu(c: SwiCase, launch, device):
    gu, dh = swiglu_inputs(c)
    errors, G = [], Guards()
    gub = G.i("gu", gu, device)
    dhb = G.i("dh", dh, device)
    hb = G.o("h", c.M * c.I, torch.bfloat16, device)
    dgub = G.o("dgu", c.M * 2 * c.I, torch.bfloat16, device)
    launch.swiglu_fwd(gub.t.view(c.M, 2 * c.I), hb.t.view(c.M, c.I))
    launch.swiglu_bwd(gub.t.view(c.M, 2 * c.I), dhb.t.view(c.M, c.I), dgub.t.view(c.M, 2 * c.I))
    G.check(errors, f"swiglu[{c.name}]")
    g, u = gu[:, 0::2].reshape(-1), gu[:, 1::2].reshape(-1)
    g64, u64, dh64 = g.double(), u.double(), dh.reshape(-1).double()
    act64, s64 = silu64(g64)
    # forward: HF's op is torch's bf16 F.silu(g) * u; it may differ from the kernel only where silu is near a tie
    want = torch.nn.functional.silu(g) * u
    near, other, tie = neighbours(act64)
    band = tie <= SILU_TIE_REL * act64.abs()
    gh = bits(hb.t.cpu())
    ok = (gh == bits(want)) | (band & ((gh == bits(rbf(near * u64))) | (gh == bits(rbf(other * u64)))))
    bad = (~ok).nonzero()[:, 0]
    if len(bad):
        ex = [(int(i), float(g[i]), float(u[i]), float(hb.t.cpu()[i]), float(want[i]),
               float(tie[i] / act64[i].abs()) if act64[i] != 0 else 0.0) for i in bad[:8]]
        errors.append(f"swiglu_fwd[{c.name}]: {len(bad)} of {g.numel()} differ from torch's bf16 F.silu(g)*u outside the "
                      f"2^-20 tie band, e.g. (index, g, u, got, torch, tie distance / |silu|) {ex}")
    flips_fwd = int((gh != bits(want)).sum()) - len(bad)
    # backward, torch's bf16 autograd chain in float64: d_up = rbf(dh * rbf(silu(g))), d_gate = rbf(rbf(dh*u) * silu'(g))
    act_c = [near, torch.where(band, other, near)]
    dup = [rbf(dh64 * a) for a in act_c]
    dact = rbf(dh64 * u64)
    dsil = s64 + g64 * s64 * (1.0 - s64)
    dgate = dact * dsil
    # the kernel's fp32 silu' (expf, one division, three products, one sum) is within 8 fp32 ulp of its terms, and the
    # fp32 sigmoid is subnormal for g < -87.3 (absolute 2^-149 per fp32 operation)
    wg = dact.abs() * (2.0 ** -21 * (s64.abs() + (g64 * s64 * (1 - s64)).abs()) + 2.0 ** -146 * (1 + g64.abs()))
    dgu = dgub.t.cpu().view(-1, 2)
    f_gate = check_band(f"swiglu_bwd[{c.name}].d_gate", dgu[:, 0], dgate, wg, errors)
    f_up = check_candidates(f"swiglu_bwd[{c.name}].d_up", dgu[:, 1], dup, errors)
    return {"errors": errors, "flips_fwd": flips_fwd, "flips_bwd": f_gate + f_up, "n": g.numel(),
            "low_gates_exact": int(((g64 <= -89) & (bits(hb.t.cpu()) == bits(want))).sum())}


# ------------------------------------------------------------------------------------------------ RMSNorm forward
NORM_TIE_REL = 2.0 ** -16       # fp32 sum of squares over H <= 8192 (<= 64 terms per thread, then two trees) is within
                                # ~2^-17 of the float64 one, rstd within half of that: x·rstd may round either way here
RSTD_REL = 2.0 ** -21           # the measured-and-derived bound on rstd itself (checked per row)
NORM_H = (8, 64, 896, 1024, 3584, 4096, 8192)


def rmsnorm_inputs(H, rows=6, seed=3):
    x = randn_bf16((rows, H), seed + H, 1.7)
    x[1] = 0                                     # all-zero row: rstd = 1/sqrt(eps), y = +-0
    x[2] = randn_bf16(H, seed + 1, 1e30)         # squares overflow fp32: HF's fp32 formula gives rstd = 0 too
    x[3] = randn_bf16(H, seed + 2, 1e-3)
    w = randn_bf16(H, seed + 5, 0.6)
    return x, w


def run_rmsnorm(H, launch, device, eps=1e-6):
    x, w = rmsnorm_inputs(H)
    rows = x.shape[0]
    errors, G = [], Guards()
    xb, wb = G.i("x", x, device), G.i("w", w, device)
    yb = G.o("y", rows * H, torch.bfloat16, device)
    rb = G.o("rstd", rows, torch.float32, device)
    launch.rmsnorm_fwd(xb.t.view(rows, H), wb.t, eps, out=yb.t.view(rows, H), rstd=rb.t)
    G.check(errors, f"rmsnorm[H={H}]")
    x64, w64 = x.double(), w.double()
    ss = (x64 * x64).sum(1, keepdim=True)
    eps32 = float(np.float32(eps))
    rstd64 = 1.0 / torch.sqrt(ss / H + eps32)
    ovf = (ss.reshape(-1) > FLT_MAX)             # the fp32 sum overflows: rstd = 1/sqrt(inf) = 0
    rstd64[ovf] = 0.0
    n64 = x64 * rstd64
    near, other, tie = neighbours(n64)
    band = tie <= NORM_TIE_REL * n64.abs()
    cands = [rbf(w64 * near), rbf(w64 * torch.where(band, other, near))]
    y = yb.t.cpu().view(rows, H)
    flips = check_candidates(f"rmsnorm[H={H}].y", y, cands, errors)
    # rows whose squares overflow: HF's own fp32 formula, bit for bit
    xf = x[ovf].float()
    hf = w * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)).to(torch.bfloat16)
    check_exact(f"rmsnorm[H={H}].overflow_rows", y[ovf], hf, errors)
    ratio = check_bound(f"rmsnorm[H={H}].rstd", rb.t.cpu().double(), rstd64.reshape(-1),
                        RSTD_REL * rstd64.reshape(-1).abs() + (rstd64.reshape(-1) == 0) * 1e-300, errors)
    return {"errors": errors, "flips": flips, "rstd_ratio": ratio}


# ------------------------------------------------------------------------------------------------ rotary tables
TABLE_TIE_REL = 2.0 ** -21      # CUDA's cosf / sinf are within 2 fp32 ulp (2^-22 relative), with full range reduction


def hf_inv_freq(d, theta):
    """HF's default rope parameters: 1 / theta^(arange(0, d, 2) / d) in fp32"""
    return 1.0 / (theta ** (torch.arange(0, d, 2, dtype=torch.int64).float() / d))


def run_rope_table(d, theta, max_pos, launch, device):
    errors = []
    inv = hf_inv_freq(d, theta)
    ib = inp(inv, device)
    snap = ib.raw.clone()
    cos, sin = launch.rope_table(ib.t, max_pos)
    if not torch.equal(ib.raw, snap):
        errors.append("rope_table: inv_freq was written")
    # HF: freqs = inv_freq @ positions in fp32 (one product per entry), cos/sin in fp32, then to bf16
    ang = f32(torch.arange(max_pos, dtype=torch.float64)[:, None] * inv.double()[None, :])
    fl = 0
    for nm, fn, got in (("cos", torch.cos, cos), ("sin", torch.sin, sin)):
        ref = fn(ang)
        fl += check_band(f"rope_table[d={d},theta={theta:g}].{nm}", got.cpu(), ref, TABLE_TIE_REL * ref.abs(), errors)
    return {"errors": errors, "flips": fl, "tables": (cos, sin)}


# ------------------------------------------------------------------------------------------------ RoPE + KV append
@dataclass(frozen=True)
class RopeCase:
    name: str
    n_h: int
    n_kv: int
    d: int
    qk_norm: bool
    B: int = 2
    S: int = 5
    pos0: int = 3
    T_max: int = 16
    kv_start: Optional[tuple] = None


def rope_fwd_cases():
    from tensorlink_b200.ml import configs as C
    cs = []
    for cfg in (C.QWEN25_05B, C.QWEN25_7B, C.QWEN3_8B, C.TINY_QWEN2, C.TINY_QWEN2_D128, C.TINY_QWEN3):
        nm = cfg.name.split("/")[-1]
        cs.append(RopeCase(nm, cfg.n_heads, cfg.n_kv_heads, cfg.head_dim, cfg.qk_norm))
        cs.append(RopeCase(nm + ".prefill0", cfg.n_heads, cfg.n_kv_heads, cfg.head_dim, cfg.qk_norm, B=1, S=9, pos0=0, T_max=9))
        cs.append(RopeCase(nm + ".leftpad", cfg.n_heads, cfg.n_kv_heads, cfg.head_dim, cfg.qk_norm, B=3, S=6, pos0=2,
                           T_max=12, kv_start=(0, 4, 7)))
    return cs


def rope_fwd_ref(q64, c64, s64):
    """HF's bf16 apply_rotary_pos_emb on one vector set: rbf(rbf(x1 c) + rbf(-x2 s)), rbf(rbf(x2 c) + rbf(x1 s))"""
    h = q64.shape[-1] // 2
    x1, x2 = q64[..., :h], q64[..., h:]
    o1 = rbf(f32(rbf(x1 * c64) + rbf(-x2 * s64)))
    o2 = rbf(f32(rbf(x2 * c64) + rbf(x1 * s64)))
    return torch.cat([o1, o2], -1)


def run_rope_fwd(c: RopeCase, tables, launch, device, eps=1e-6, seed=5):
    cos, sin = (t.cpu() for t in tables)
    heads = c.n_h + 2 * c.n_kv
    n_tok = c.B * c.S
    qkv = randn_bf16((n_tok, heads * c.d), seed + heads + c.d, 1.3)
    qn, kn = randn_bf16(c.d, seed + 1, 0.5) + 1.0, randn_bf16(c.d, seed + 2, 0.5) + 1.0
    qn, kn = qn.to(torch.bfloat16), kn.to(torch.bfloat16)
    errors, G = [], Guards()
    qb = G.i("qkv", qkv, device)
    qnb, knb = (G.i("q_norm", qn, device), G.i("k_norm", kn, device)) if c.qk_norm else (None, None)
    cb, sb = G.i("cos", cos, device), G.i("sin", sin, device)
    pb = G.i("pos0", torch.tensor([c.pos0], dtype=torch.int32), device)
    ksb = G.i("kv_start", torch.tensor(c.kv_start, dtype=torch.int32), device) if c.kv_start else None
    qo = G.o("q_out", n_tok * c.n_h * c.d, torch.bfloat16, device)
    cache_n = c.B * c.n_kv * c.T_max * c.d
    kc = out(cache_n, torch.bfloat16, device)     # slots outside [pos0, pos0+S) must keep their sentinel
    vc = out(cache_n, torch.bfloat16, device)
    launch.rope_kv_fwd(qb.t.view(n_tok, -1), qo.t.view(n_tok, -1), kc.t.view(c.B, c.n_kv, c.T_max, c.d),
                       vc.t.view(c.B, c.n_kv, c.T_max, c.d), pb.t, cb.t.view(cos.shape), sb.t.view(sin.shape),
                       qnb.t if qnb else None, knb.t if knb else None, eps, c.S, c.n_h, c.n_kv, c.d,
                       kv_start=ksb.t if ksb else None)
    G.check(errors, f"rope_fwd[{c.name}]")
    for nm, b in (("k_cache", kc), ("v_cache", vc)):
        if b.pads_changed():
            errors.append(f"rope_fwd[{c.name}]: guard elements around {nm} were written")
    x = qkv.double().view(c.B, c.S, heads, c.d)
    pos = c.pos0 + torch.arange(c.S)
    ks = torch.tensor(c.kv_start or (0,) * c.B)
    rpos = (pos[None, :] - ks[:, None]).clamp_min(0)                                   # [B, S]
    half = c.d // 2
    cc = cos.double()[rpos][:, :, None, :]                                              # [B, S, 1, half]
    ss = sin.double()[rpos][:, :, None, :]
    qk = x[:, :, :c.n_h + c.n_kv]
    flips = 0
    if not c.qk_norm:
        # HF bit for bit, in torch's own bf16 ops
        xb = qk.to(torch.bfloat16)
        cb16, sb16 = torch.cat([cc, cc], -1).to(torch.bfloat16), torch.cat([ss, ss], -1).to(torch.bfloat16)
        rot = torch.cat([-xb[..., half:], xb[..., :half]], -1)
        want = [xb * cb16 + rot * sb16]
    else:
        # Qwen3 q/k-norm: fp32 rstd, so each normalised element may flip where it lies within 2^-16 of a tie: every
        # combination of the pair's (x1, x2) candidates is allowed
        w = torch.cat([qn.double().expand(c.n_h, c.d), kn.double().expand(c.n_kv, c.d)])
        rstd = 1.0 / torch.sqrt((qk * qk).mean(-1, keepdim=True) + float(np.float32(eps)))
        n64 = qk * rstd
        near, other, tie = neighbours(n64)
        alt = torch.where(tie <= NORM_TIE_REL * n64.abs(), other, near)
        y0, y1 = rbf(w * near), rbf(w * alt)
        want = []
        for a in (y0, y1):
            for b in (y0, y1):
                v = torch.cat([a[..., :half], b[..., half:]], -1)
                want.append(rope_fwd_ref(v, cc, ss))
    got_q = qo.t.cpu().view(c.B, c.S, c.n_h, c.d)
    got_k = kc.t.cpu().view(c.B, c.n_kv, c.T_max, c.d)[:, :, c.pos0:c.pos0 + c.S].permute(0, 2, 1, 3)
    got = torch.cat([got_q, got_k], 2)
    if c.qk_norm:
        flips = check_candidates(f"rope_fwd[{c.name}].qk", got, [w_.double() for w_ in want], errors)
    else:
        check_exact(f"rope_fwd[{c.name}].qk", got, want[0], errors)
    got_v = vc.t.cpu().view(c.B, c.n_kv, c.T_max, c.d)[:, :, c.pos0:c.pos0 + c.S].permute(0, 2, 1, 3)
    check_exact(f"rope_fwd[{c.name}].v", got_v, qkv.view(c.B, c.S, heads, c.d)[:, :, c.n_h + c.n_kv:], errors)
    for nm, b in (("k_cache", kc), ("v_cache", vc)):
        full = b.raw.cpu()[PAD:PAD + cache_n].view(c.B, c.n_kv, c.T_max, c.d).clone()
        full[:, :, c.pos0:c.pos0 + c.S] = BF16_SENTINEL
        if (full != BF16_SENTINEL).any():
            errors.append(f"rope_fwd[{c.name}]: {nm} slots outside [pos0, pos0+S) were written")
    return {"errors": errors, "flips": flips}


# ------------------------------------------------------------------------------------------------ RoPE backward
@dataclass(frozen=True)
class RopeBwdCase:
    name: str
    n_h: int
    n_kv: int
    d: int
    B: int
    S: int
    T_pad: int = 3              # T_max = S + T_pad; rows S..T_max-1 of dk / dv hold NaN

    @property
    def n_rep(self):
        return self.n_h // self.n_kv


def rope_bwd_cases():
    return [RopeBwdCase("0.5B.S63", 14, 2, 64, 2, 63),          # n_rep 7, d 64
            RopeBwdCase("7B.S65", 28, 4, 128, 1, 65),           # n_rep 7, d 128
            RopeBwdCase("8B.S64", 32, 8, 128, 1, 64),           # n_rep 4
            RopeBwdCase("rep1.S1", 4, 4, 64, 3, 1),
            RopeBwdCase("rep2.S700", 4, 2, 128, 1, 700),
            RopeBwdCase("rep8.S65", 16, 2, 64, 2, 65),
            RopeBwdCase("rep8.d128.S63", 8, 1, 128, 2, 63)]


def rope_bwd_inputs(c: RopeBwdCase, leg, seed=9):
    n_tok, T = c.B * c.S, c.S + c.T_pad
    sh_q, sh_kv = (n_tok, c.n_h, c.d), (c.B, c.n_h, T, c.d)
    if leg == "exact":      # integer partials in [-8, 8]: the fp32 sum of <= 8 partials is exact, every rotation product too
        mk = lambda sh, s: torch.randint(-8, 9, sh, generator=_gen(s)).to(torch.bfloat16)
    else:
        mk = lambda sh, s: randn_bf16(sh, s, 1.0)
    dq = mk(sh_q, seed)
    dk, dv = mk(sh_kv, seed + 1), mk(sh_kv, seed + 2)
    dk[:, :, c.S:] = float("nan")
    dv[:, :, c.S:] = float("nan")
    return dq, dk, dv


def rope_bwd_ref(c: RopeBwdCase, dq, dk, dv, cos, sin):
    """float64 (value, |terms| for the rounding bound) of dqkv [n_tok, heads, d]"""
    S, half = c.S, c.d // 2
    g = lambda t: t.double()[:, :, :S].view(c.B, c.n_kv, c.n_rep, S, c.d)
    sk, sv = g(dk).sum(2), g(dv).sum(2)                              # [B, n_kv, S, d]
    ak = g(dk).abs().sum(2)
    tok = lambda t: t.permute(0, 2, 1, 3).reshape(c.B * S, c.n_kv, c.d)
    dqk = torch.cat([dq.double(), tok(sk)], 1)
    aqk = torch.cat([dq.double().abs(), tok(ak)], 1)
    pos = torch.arange(c.B * S) % S
    cc, ss = cos.double()[pos][:, None, :], sin.double()[pos][:, None, :]
    d1, d2 = dqk[..., :half], dqk[..., half:]
    a1, a2 = aqk[..., :half], aqk[..., half:]
    val = torch.cat([d1 * cc + d2 * ss, d2 * cc - d1 * ss], -1)
    mag = torch.cat([a1 * cc.abs() + a2 * ss.abs(), a2 * cc.abs() + a1 * ss.abs()], -1)
    return torch.cat([val, tok(sv)], 1), torch.cat([mag, tok(g(dv).abs().sum(2))], 1)


def run_rope_bwd(c: RopeBwdCase, leg, tables, launch, device):
    cos, sin = (t.cpu() for t in tables)
    dq, dk, dv = rope_bwd_inputs(c, leg)
    n_tok, heads = c.B * c.S, c.n_h + 2 * c.n_kv
    errors, G = [], Guards()
    qb, kb, vb = G.i("dq", dq, device), G.i("dk", dk, device), G.i("dv", dv, device)
    cb, sb = G.i("cos", cos, device), G.i("sin", sin, device)
    ob = G.o("dqkv", n_tok * heads * c.d, torch.bfloat16, device)
    launch.rope_kv_bwd(qb.t.view(dq.shape), kb.t.view(dk.shape), vb.t.view(dv.shape), ob.t.view(n_tok, heads * c.d),
                       cb.t.view(cos.shape), sb.t.view(sin.shape), c.S, c.n_h, c.n_kv, c.d)
    G.check(errors, f"rope_bwd[{c.name}/{leg}]")
    val, mag = rope_bwd_ref(c, dq, dk, dv, cos, sin)
    got = ob.t.cpu().view(n_tok, heads, c.d)
    ratio = 0.0
    if leg == "exact":
        # the rotation's fp32 result is the exact value rounded once to fp32 (whether or not the compiler fuses it)
        check_exact(f"rope_bwd[{c.name}/exact]", got, rbf(f32(val)), errors)
    else:
        # one bf16 ulp, plus 2^-20 of the summed magnitudes (<= 7 fp32 additions of partials and the rotation)
        ratio = check_bound(f"rope_bwd[{c.name}/round]", got, val, ulp_bf16(val) + 2.0 ** -20 * mag, errors)
    return {"errors": errors, "ratio": ratio}


# ------------------------------------------------------------------------------------------------ cross-entropy dlogits
@dataclass(frozen=True)
class CeCase:
    name: str
    V: int
    scale: float = 1.0 / 37


def ce_cases():
    return [CeCase("V8", 8), CeCase("V1000", 1000), CeCase("V151936", 151936, 0.125)]


def ce_inputs(c: CeCase, seed=21):
    M = 7
    logits = randn_bf16((M, c.V), seed + c.V, 2.5)
    labels = torch.tensor([0, c.V - 1, c.V - 3, -100, 1 % c.V, c.V // 2, c.V - 8], dtype=torch.int64)
    logits[4, 1 % c.V] = float(logits[4].float().max()) + 90.0          # one logit 90 above the rest (p_max ~ 1)
    logits[5].mul_(0.01)
    return logits, labels


def ce_ref(logits, labels, scale):
    x = logits.double()
    p = torch.softmax(x, -1)
    oh = torch.zeros_like(p)
    valid = (labels >= 0) & (labels < x.shape[1])
    oh[valid.nonzero()[:, 0], labels[valid]] = 1.0
    return (p - oh) * scale * valid[:, None], p.max(-1).values, valid


def run_ce(c: CeCase, launch, device):
    logits, labels = ce_inputs(c)
    M = logits.shape[0]
    errors, G = [], Guards()
    lb, yb = G.i("logits", logits, device), G.i("labels", labels, device)
    db = G.o("dlogits", M * c.V, torch.bfloat16, device)
    loss, nv = torch.zeros(1, dtype=torch.float32, device=device), torch.zeros(1, dtype=torch.int32, device=device)
    launch.ce_fwd_bwd(lb.t.view(M, c.V), yb.t, loss, nv, db.t.view(M, c.V), c.scale)
    G.check(errors, f"ce[{c.name}]")
    ref, pmax, valid = ce_ref(logits, labels, c.scale)
    # one bf16 ulp + 2^-20·p_max·scale (fp32 exp and the row sum's rounding, relative to the row's largest term) +
    # 2^-126·scale (exp of a logit ~90 below the max is an fp32 subnormal)
    bound = ulp_bf16(ref) + (2.0 ** -20 * pmax[:, None] + 2.0 ** -126) * c.scale
    got = db.t.cpu().view(M, c.V)
    ratio = check_bound(f"ce[{c.name}].dlogits", got, ref, bound, errors)
    if (bits(got[~valid]) != 0).any():
        errors.append(f"ce[{c.name}]: an ignored row is not exactly +0")
    # the trainer's call: dlogits = logits, in place; it must equal the out-of-place result bit for bit
    ib = inp(logits, device)
    loss2, nv2 = torch.zeros_like(loss), torch.zeros_like(nv)
    launch.ce_fwd_bwd(ib.t.view(M, c.V), yb.t, loss2, nv2, ib.t.view(M, c.V), c.scale)
    if ib.pads_changed():
        errors.append(f"ce[{c.name}]: the in-place call wrote outside the logits")
    check_exact(f"ce[{c.name}].in_place", ib.t.cpu().view(M, c.V), got, errors)
    if not torch.equal(loss2.cpu(), loss.cpu()):
        errors.append(f"ce[{c.name}]: in-place loss {float(loss2)} != out-of-place {float(loss)}")
    return {"errors": errors, "ratio": ratio}


# ------------------------------------------------------------------------------------------------ embedding
def run_embed(H, n_tok, launch, device, vocab=50, seed=31):
    table = randn_bf16((vocab, H), seed + H)
    ids = torch.randint(0, vocab, (n_tok,), generator=_gen(seed + n_tok))
    ids[::7] = -1                                # out of range: row 0, as documented (callers validate on the host)
    ids[3::11] = vocab
    ids[5::13] = -(2 ** 40)
    ids[0] = vocab - 1
    errors, G = [], Guards()
    ib, tb = G.i("ids", ids, device), G.i("table", table, device)
    ob = G.o("out", n_tok * H, torch.bfloat16, device)
    launch.embed_fwd(ib.t, tb.t.view(vocab, H), ob.t.view(n_tok, H))
    G.check(errors, f"embed[H={H},n={n_tok}]")
    want = table[torch.where((ids >= 0) & (ids < vocab), ids, torch.zeros_like(ids))]
    check_exact(f"embed[H={H},n={n_tok}]", ob.t.cpu().view(n_tok, H), want, errors)
    return {"errors": errors}


# ------------------------------------------------------------------------------------------------ gradient commits
COMMIT_N = (8, 4096, 2 ** 20 + 8)
COMMIT_N_RAGGED = (1, 7, 4099, 2 ** 20 + 3)      # the fp32-source entry points take any n


def tie_f32(n, seed):
    """fp32 values whose low 16 bits sit on, just below and just above a bf16 rounding tie (and random ones)"""
    r = torch.randn(n, generator=_gen(seed), dtype=torch.float32)
    b = r.view(torch.int32) & ~0xFFFF
    low = torch.tensor([0x8000, 0x7FFF, 0x8001, 0x0000, 0xFFFF], dtype=torch.int32)
    sel = torch.arange(n) % 6
    lowbits = torch.where(sel < 5, low[sel.clamp_max(4)], r.view(torch.int32) & 0xFFFF)
    return (b | lowbits).view(torch.float32)


def run_commit(kind, n, accumulate, launch, device, seed=41):
    """kind: add | scale_bf16 | scale_f32 | f32_to_bf16 | alias (commit_head's scale_add(x, x, s, accumulate=False))"""
    errors, G = [], Guards()
    s = 0.3 if kind != "alias" else 1.0 / 24
    s64 = float(np.float32(s))
    name = f"{kind}[n={n},acc={int(accumulate)}]"
    if kind == "scale_f32":
        a0, b0 = torch.randn(n, generator=_gen(seed)), torch.randn(n, generator=_gen(seed + 1))
        bb = G.i("b", b0, device)
        ab = G.o("a", n, torch.float32, device, a0)
        launch.scale_add(ab.t, bb.t, s, accumulate)
        G.check(errors, name)
        want = f32(s64 * b0.double() + (a0.double() if accumulate else 0.0))   # fmaf: one fp32 rounding
        if not torch.equal(ab.t.cpu().view(torch.int32), want.float().view(torch.int32)):
            bad = int((ab.t.cpu().view(torch.int32) != want.float().view(torch.int32)).sum())
            errors.append(f"{name}: {bad} of {n} differ from fp32(s·b + a)")
        return {"errors": errors}
    if kind == "f32_to_bf16":
        src = tie_f32(n, seed)
        d0 = randn_bf16(n, seed + 1, 0.01)
        sb = G.i("src", src, device)
        db = G.o("dst", n, torch.bfloat16, device, d0)
        launch.f32_to_bf16_accum(sb.t, db.t, accumulate)
        G.check(errors, name)
        want = rbf(f32(src.double() + (d0.double() if accumulate else 0.0)))
        check_exact(name, db.t, want, errors)
        return {"errors": errors}
    a0 = tie_f32(n, seed).to(torch.bfloat16)
    b0 = randn_bf16(n, seed + 1)
    if kind == "alias":
        ab = G.o("a", n, torch.bfloat16, device, b0)
        launch.scale_add(ab.t, ab.t, s, False)
        G.check(errors, name)
        check_exact(name, ab.t, rbf(f32(s64 * b0.double())), errors)
        return {"errors": errors}
    bb = G.i("b", b0, device)
    ab = G.o("a", n, torch.bfloat16, device, a0)
    if kind == "add":
        launch.add_inplace(ab.t, bb.t)
        want = rbf(f32(a0.double() + b0.double()))
    else:
        launch.scale_add(ab.t, bb.t, s, accumulate)
        want = rbf(f32(s64 * b0.double() + (a0.double() if accumulate else 0.0)))   # fmaf, then bf16
    G.check(errors, name)
    check_exact(name, ab.t, want, errors)
    return {"errors": errors}


# ------------------------------------------------------------------------------------------------ AdamW
ADAM_N = (1, 7, 8, 9, 4099, 2 ** 20 + 3)
ADAM_STEPS = (1, 2, 10, 1000, 100000)
ADAM_P_TIE = 2.0 ** -16         # relative to |p| + |update|: the fp32 update chain (a handful of roundings, ~2^-21)
ADAM_MV_ULP = 4                 # m, v: fp32 ulps of the larger of their two terms (the recurrence may cancel)


@dataclass(frozen=True)
class AdamCfg:
    name: str
    decoupled: bool
    wd: float
    lr: float = 1e-3
    b1: float = 0.9
    b2: float = 0.999
    eps: float = 1e-8


ADAM_CFGS = (AdamCfg("adam", False, 0.0), AdamCfg("adam_wd", False, 0.01), AdamCfg("adamw", True, 0.0),
             AdamCfg("adamw_wd", True, 0.1))


_LIBM = None


def host_bias_corrections(b1, b2, step):
    """(bc1, sqrt(bc2)) as tl_adamw_step forms them on the host: fp32 ``1 - powf(beta, step)`` with the C library's powf.
    torch.optim.Adam forms them in double; the fp32 ones differ by up to 2^-14 relative at small steps (1 - beta2^t
    cancels), which is a property of the kernel's interface, so the reference takes them as given."""
    global _LIBM
    if _LIBM is None:
        import ctypes
        import ctypes.util
        _LIBM = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
        _LIBM.powf.restype, _LIBM.powf.argtypes = ctypes.c_float, [ctypes.c_float, ctypes.c_float]
    F = np.float32
    bc1 = F(1) - F(_LIBM.powf(F(b1), F(step)))
    bc2s = np.sqrt(F(1) - F(_LIBM.powf(F(b2), F(step))))
    return float(bc1), float(bc2s)


def adam_ref(p, g, m, v, a: AdamCfg, step):
    """float64 torch.optim.Adam/AdamW on the fp32 hyperparameters and bias corrections the kernel receives;
    (p', m', v', m and v term scales, update, p before the update)"""
    F = lambda x: float(np.float32(x))
    lr, b1, b2, eps, wd = F(a.lr), F(a.b1), F(a.b2), F(a.eps), F(a.wd)
    p, g, m, v = p.double(), g.double(), m.double(), v.double()
    if wd:
        if a.decoupled:
            p = p * (1 - lr * wd)
        else:
            g = g + wd * p
    m1 = b1 * m + (1 - b1) * g
    v1 = b2 * v + (1 - b2) * g * g
    bc1, bc2s = host_bias_corrections(a.b1, a.b2, step)
    upd = (lr / bc1) * m1 / (torch.sqrt(v1) / bc2s + eps)
    sm = torch.maximum((b1 * m).abs(), ((1 - b1) * g).abs())
    sv = torch.maximum((b2 * v).abs(), ((1 - b2) * g * g).abs())
    return p - upd, m1, v1, sm, sv, upd, p


def adam_state(n, seed, zero_grad=False):
    p = randn_bf16(n, seed, 0.05)
    g = torch.zeros(n, dtype=torch.bfloat16) if zero_grad else randn_bf16(n, seed + 1, 0.02)
    m = torch.randn(n, generator=_gen(seed + 2)) * (1e-12 if zero_grad else 1e-3)
    v = torch.zeros(n) if zero_grad else torch.rand(n, generator=_gen(seed + 3)) * 1e-4
    return p, g, m, v


def run_adam(n, a: AdamCfg, steps, launch, device, seed=51, spans=None, zero_grad=False, lr_zero=False):
    """``steps`` in order, each checked alone from the kernel's own state (error does not compound); ``spans``: the
    [a, e) pieces StageAdam hands over, called one by one at their offsets inside one arena"""
    if lr_zero:
        a = AdamCfg(a.name + ".lr0", a.decoupled, a.wd, lr=0.0)
    p0, g0, m0, v0 = adam_state(n, seed + n, zero_grad)
    errors, G = [], Guards()
    gb = G.i("g", g0, device)
    pb = G.o("p", n, torch.bfloat16, device, p0)
    mb = G.o("m", n, torch.float32, device, m0)
    vb = G.o("v", n, torch.float32, device, v0)
    ratio_p, ratio_mv, flips = 0.0, 0.0, 0
    name = f"adam[{a.name},n={n}{',spans' if spans else ''}{',zero_grad' if zero_grad else ''}]"
    for t in steps:
        p, m, v = pb.t.cpu().clone(), mb.t.cpu().clone(), vb.t.cpu().clone()
        for s0, s1 in (spans or [(0, n)]):
            launch.adamw_step(pb.t[s0:s1], gb.t[s0:s1], mb.t[s0:s1], vb.t[s0:s1], a.lr, a.b1, a.b2, a.eps, a.wd, t,
                              a.decoupled)
        G.check(errors, f"{name}@{t}")
        if lr_zero:
            check_exact(f"{name}@{t}.p", pb.t, p, errors)
            continue
        p1, m1, v1, sm, sv, upd, pw = adam_ref(p, g0, m, v, a, t)
        ratio_mv = max(ratio_mv, check_bound(f"{name}@{t}.m", mb.t.cpu().double(), m1, ADAM_MV_ULP * ulp_f32(sm) + 1e-45, errors),
                       check_bound(f"{name}@{t}.v", vb.t.cpu().double(), v1, ADAM_MV_ULP * ulp_f32(sv) + 1e-45, errors))
        flips += check_band(f"{name}@{t}.p", pb.t, p1, ADAM_P_TIE * (pw.abs() + upd.abs()), errors)
        ratio_p = max(ratio_p, check_bound(f"{name}@{t}.p_ulp", pb.t.cpu().double(), p1, ulp_bf16(p1), errors))
    return {"errors": errors, "ratio_p": ratio_p, "ratio_mv": ratio_mv, "flips": flips}


def stage_adam_spans(sizes, tail):
    """StageAdam's cut of an arena: layer spans [a, e) rounded up to 128 elements, in reverse order (the backward finishes
    the last layer first), then the rest (embedding, final norm, head) up to the arena's ragged end"""
    spans, a = [], 0
    for s in sizes:
        e = a + (s + 127) // 128 * 128
        spans.append((a, e))
        a = e
    return list(reversed(spans)) + [(a, a + tail)], a + tail


# ------------------------------------------------------------------------------------------------ sampling: Philox
M32 = 0xFFFFFFFF
PHILOX_KAT = (((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
              ((M32,) * 4, (M32, M32), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)))   # Random123 kat_vectors


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al., SC'11) on uint64 numpy arrays holding 32-bit words; the kernel's philox_round and
    key schedule (csrc/sample.cu)"""
    c0, c1, c2, c3 = (np.asarray(x, dtype=np.uint64) & M32 for x in ctr)
    k0, k1 = (np.asarray(x, dtype=np.uint64) & M32 for x in key)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & np.uint64(M32), (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & np.uint64(M32)
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & np.uint64(M32), (k1 + np.uint64(0xBB67AE85)) & np.uint64(M32)
    return c0, c1, c2, c3


def philox_u(seed, row, counters):
    """the kernel's uniform: counter block (counter, row, 0x5eed5eed, 0), key = seed; u = (c0 >> 8) / 2^24"""
    counters = np.asarray(counters, dtype=np.uint64)
    c0, *_ = philox4x32_10((counters, np.full_like(counters, row), np.full_like(counters, 0x5EED5EED), np.zeros_like(counters)),
                           (seed & M32, seed >> 32))
    return (c0 >> np.uint64(8)).astype(np.float64) / 16777216.0


# ------------------------------------------------------------------------------------------------ sampling: model
EXP_REL = 2.0 ** -21            # __expf / expf: 2 fp32 ulp of the result (ex2.approx, or the IEEE-accurate expf)
ARG_REL = 2.0 ** -24            # one fp32 rounding of an argument is |x|·2^-24 in the exponent; __expf adds one for x·log2e


def _bf16_key(b):
    b = b.astype(np.int64) & 0xFFFF
    return np.where(b & 0x8000, (~b) & 0xFFFF, b | 0x8000)


@dataclass
class RowModel:
    kept: np.ndarray            # bool [V]
    w: np.ndarray               # float64 weights (0 outside kept)
    err: np.ndarray             # float64 bound on each weight's error (same units)
    C: np.ndarray               # cumulative kept weight in index order
    Zk: float                   # the mass the target scales (tl_sample: Z_kept of the bins; _proc: W)
    proc: bool
    pinned: bool                # no top-p boundary inside its error band
    banned_all: bool = False


def sample_row_model(logits_row_bf16: torch.Tensor, temperature, top_k, top_p, proc=False, present=None, banned=None,
                     penalty=1.0, fault=None) -> RowModel:
    """The kept set and the weights of one row as the kernel's documented rules define them, in float64."""
    V = logits_row_bf16.numel()
    it = float(np.float32(1.0) / np.float32(temperature))
    x = logits_row_bf16.float().numpy().astype(np.float32)
    if proc:
        if present is not None:
            pen = np.float32(penalty)
            xp = np.where(x < 0, x * pen, x / pen).astype(np.float32)
            x = np.where(present, xp, x)
        if banned is not None:
            x = np.where(banned, np.float32(-np.inf), x)
        x = np.where(x == 0, np.float32(0), x)          # -0 and +0 share a key
        if not np.isfinite(x).any() or np.max(x) == -np.inf:
            return RowModel(np.zeros(V, bool), np.zeros(V), np.zeros(V), np.zeros(V), 0.0, True, True, banned_all=True)
        key = x.view(np.uint32).astype(np.int64)
        key = np.where(key & 0x80000000, (~key) & 0xFFFFFFFF, key | 0x80000000)
        x_max = float(np.float32(np.max(x)) * np.float32(it))
    else:
        key = _bf16_key(logits_row_bf16.view(torch.int16).numpy())
        x_max = float(np.float32(x[np.argmax(key)]) * np.float32(it))
    x64 = x.astype(np.float64)
    k_key = 0
    if 0 < top_k < V:
        k_key = np.sort(key)[::-1][top_k - 1]
    kk = key >= k_key
    arg = x64 * it - x_max
    with np.errstate(over="ignore", invalid="ignore"):
        w = np.where(kk, np.exp(np.where(kk, arg, 0.0)), 0.0)
    rel = EXP_REL + ARG_REL * (2 * np.abs(arg) + np.abs(x64 * it))
    rel = np.where(np.isfinite(rel), rel, 0.0)
    if proc:
        w = np.floor(w * 2.0 ** 40)
        err = w * rel + 1.0                              # fixed point: one truncation per token
    else:
        w = np.where(w < 2.0 ** -126, 0.0, w)            # __expf flushes subnormal results to zero
        err = w * rel + 2.0 ** -126
    pinned = True
    p_key = k_key
    if top_p < 1.0:
        uk, inv = np.unique(np.where(kk, key, -1), return_inverse=True)
        mass = np.bincount(inv, weights=w)[::-1]         # per distinct key, descending
        emass = np.bincount(inv, weights=np.where(kk, err, 0.0))[::-1]
        keys_desc = uk[::-1]
        valid = keys_desc >= 0
        mass, emass, keys_desc = mass[valid], emass[valid], keys_desc[valid]
        above = np.concatenate([[0.0], np.cumsum(mass)[:-1]])
        Z, EZ = mass.sum(), emass.sum()
        if proc:
            T = math.ceil(float(np.float32(top_p)) * Z)
            idx = int(np.nonzero(above + mass >= T)[0][0])          # above < T <= above + h
            band = EZ * (1 + float(np.float32(top_p))) + 2
            pinned = (T - above[idx] > band) and (above[idx] + mass[idx] - T > band)
        else:
            lim = float(np.float32(top_p)) * Z
            keep = above < lim
            idx = int(np.nonzero(keep)[0][-1])
            margin = np.abs(above - lim)
            pinned = bool(margin.min() > 2 * EZ) if len(margin) else True
        if fault == "top_p_low":
            idx = min(idx + 1, len(keys_desc) - 1)                  # one bin too many kept
        p_key = keys_desc[idx]
        Zk = float(mass[:idx + 1].sum())
    kept = key >= p_key
    w = np.where(kept, w, 0.0)
    err = np.where(kept, err, 0.0)
    C = np.cumsum(w)
    if top_p >= 1.0:
        Zk = float(w.sum())
    if proc:
        Zk = float(C[-1])
    return RowModel(kept, w, err, C, Zk, proc, pinned)


def model_draws(rm: RowModel, u: np.ndarray, fault=None):
    """(token, allowed lo, allowed hi, in band) per uniform u: the float64 inverse CDF in index order, with the fallback
    to the last kept token; [lo, hi] are the kept tokens whose CDF interval lies within the error band of the target"""
    if rm.banned_all:
        z = np.zeros(len(u), np.int64)
        return z, z, z, np.zeros(len(u), bool)
    last = int(np.nonzero(rm.kept)[0][-1])
    E = float(rm.err.sum())
    if rm.proc:
        W = rm.Zk
        t = np.minimum(W - 1, np.floor(u * W))
        b = u * E + E + 2
    else:
        t = u * rm.Zk
        b = u * E + E
    tok = np.searchsorted(rm.C, t, side="right")
    if fault == "next_token":                # `target <= c` walked one token on: the pick lands past the CDF boundary
        tok = np.searchsorted(rm.C, rm.C[np.minimum(tok, len(rm.C) - 1)], side="right")
    lo = np.searchsorted(rm.C, t - b, side="right")
    hi = np.searchsorted(rm.C, t + b, side="right")
    tok, lo, hi = (np.where(a >= len(rm.C), last, a) for a in (tok, lo, hi))
    return tok, lo, np.minimum(hi, last), lo != hi


def check_draws(name, got, rm: RowModel, u, errors):
    """every draw equals the model's token, or (inside the band) another kept token of positive weight within it"""
    tok, lo, hi, band = model_draws(rm, u)
    got = np.asarray(got, dtype=np.int64)
    ok = got == tok
    ins = band & (got >= lo) & (got <= hi)
    ins &= rm.kept[np.clip(got, 0, len(rm.kept) - 1)] & (rm.w[np.clip(got, 0, len(rm.w) - 1)] > 0) | rm.banned_all
    bad = np.nonzero(~(ok | ins))[0]
    if len(bad):
        ex = [(int(i), int(got[i]), int(tok[i])) for i in bad[:5]]
        errors.append(f"{name}: {len(bad)} of {len(got)} draws differ from the model, e.g. (draw, got, model) {ex}")
    return int(band.sum())


@dataclass(frozen=True)
class SampleCase:
    name: str
    V: int
    M: int
    temperature: float
    top_k: int = 0
    top_p: float = 1.0
    proc: bool = False
    penalty: float = 1.0
    n_ban: int = 0              # the first n_ban EOS ids of each row (min_new_tokens), row M-1: every token if V <= 8
    logit_scale: float = 2.0
    tie_k: bool = False         # top_k lands inside a group of equal logits


def sample_cases():
    return [SampleCase("V1", 1, 2, 1.0),
            SampleCase("V7", 7, 3, 1.0),
            SampleCase("V48.t20", 48, 9, 20.0),
            SampleCase("V48.k1", 48, 4, 1.0, top_k=1),
            SampleCase("V48.ktie", 48, 4, 1.0, top_k=6, tie_k=True),
            SampleCase("V48.p", 48, 4, 1.0, top_p=0.7),
            SampleCase("V1000.t005", 1000, 5, 0.05),
            SampleCase("V1000.k_ge_V", 1000, 3, 1.0, top_k=1000, logit_scale=6.0),
            SampleCase("V1000.k40p", 1000, 3, 1.0, top_k=40, top_p=0.8),
            SampleCase("V151936.k50", 151936, 2, 1.0, top_k=50),
            SampleCase("V151936.t005p", 151936, 2, 0.05, top_p=0.9),
            SampleCase("proc.V48", 48, 4, 1.0, proc=True, penalty=1.3, n_ban=3),
            SampleCase("proc.V7.banned", 7, 3, 1.0, proc=True, penalty=1.3, n_ban=7),
            SampleCase("proc.V1000.kp", 1000, 3, 0.7, top_k=30, top_p=0.85, proc=True, penalty=1.2, n_ban=2),
            SampleCase("proc.V151936.k", 151936, 2, 1.0, top_k=64, proc=True, penalty=1.5, n_ban=1),
            SampleCase("proc.V1000.t20", 1000, 2, 20.0, top_k=100, proc=True, penalty=2.0)]


N_DRAWS = 2000
SEED = 0x9E3779B97F4A7C15


def sample_inputs(c: SampleCase, seed=61):
    x = torch.randn(c.M, c.V, generator=_gen(seed + c.V), dtype=torch.float64) * c.logit_scale
    if c.tie_k:
        x[:, :] = torch.minimum(x, torch.tensor(3.0))
        x[:, :10] = 3.0                                  # ten tokens share the top value; top_k = 6 cuts inside them
    logits = x.to(torch.bfloat16)
    counters = torch.tensor([1000 * m + 17 * (m % 3) for m in range(c.M)], dtype=torch.int32)   # distinct per row
    prompt = torch.randint(0, c.V, (c.M, 5), generator=_gen(seed + 1))
    eos = list(range(min(c.n_ban, 8)))
    return logits, counters, prompt, eos


def proc_row_inputs(c: SampleCase, prompt, eos, m):
    present = np.zeros(c.V, bool)
    present[prompt[m].numpy()] = True
    banned = np.zeros(c.V, bool)
    banned[eos] = True
    return present, banned


def case_models(c: SampleCase, logits, prompt, eos, fault=None):
    models = []
    for m in range(c.M):
        if c.proc:
            present, banned = proc_row_inputs(c, prompt, eos, m)
            models.append(sample_row_model(logits[m], c.temperature, c.top_k, c.top_p, True, present,
                                           banned if eos else None, c.penalty, fault=fault))
        else:
            models.append(sample_row_model(logits[m], c.temperature, c.top_k, c.top_p, fault=fault))
    return models


def run_sample(c: SampleCase, launch, device):
    logits, counters, prompt, eos = sample_inputs(c)
    errors = []
    models = case_models(c, logits, prompt, eos)
    for m, rm in enumerate(models):
        if not rm.pinned:
            errors.append(f"sample[{c.name}] row {m}: a top-p boundary lies inside its error band (case not pinned)")
    ids = launch.sample_many(c, logits, counters, prompt, eos, N_DRAWS)      # [N, M]
    band, total = 0, 0
    for m in range(c.M):
        u = philox_u(SEED, m, np.arange(N_DRAWS, dtype=np.uint64) + int(counters[m]))
        band += check_draws(f"sample[{c.name}] row {m}", ids[:, m], models[m], u, errors)
        total += N_DRAWS
    return {"errors": errors, "band": band, "draws": total}


# ------------------------------------------------------------------------------------------------ launchers
class NativeLaunch:
    """tensorlink_b200.native, plus the repeated sampler call of run_sample"""

    def __init__(self, nat):
        self.nat = nat

    def __getattr__(self, k):
        return getattr(self.nat, k)

    def sample_many(self, c: SampleCase, logits, counters, prompt, eos, n):
        nat = self.nat
        lg = logits.cuda()
        ids = torch.empty(c.M, dtype=torch.int64, device="cuda")
        ctr = counters.cuda().clone()
        out = []
        if not c.proc:
            ws = torch.empty(nat.sample_ws(c.M), dtype=torch.uint8, device="cuda")
            for _ in range(n):
                nat.sample(lg, ids, ctr, ws, c.temperature, c.top_k, c.top_p, SEED)
                out.append(ids.clone())
        else:
            L, V = 64, c.V
            log = torch.zeros(c.M, L, dtype=torch.int32, device="cuda")
            ln = torch.zeros(c.M, dtype=torch.int32, device="cuda")
            bt = torch.zeros(c.M, (V + 31) // 32, dtype=torch.int32, device="cuda")
            ws = torch.empty(nat.logits_proc_ws(c.M, V), dtype=torch.uint8, device="cuda")
            nat.history_fill(prompt.cuda().contiguous(), log, ln, bt, V)
            ln0, bt0 = ln.clone(), bt.clone()
            params = nat.lp_params(c.penalty, 0, 100 if eos else 0, prompt.shape[1], eos).cuda()
            flags = nat.LP_BAN if eos else 0
            for _ in range(n):
                nat.sample_proc(lg, ids, log, ln, bt, params, ctr, ws, c.temperature, c.top_k, c.top_p, SEED, flags)
                out.append(ids.clone())
                ln.copy_(ln0)             # every draw sees the same history (the kernel appends its pick)
                bt.copy_(bt0)
        got = ctr.cpu()
        if not torch.equal(got, counters + n):
            raise AssertionError(f"counters advanced to {got.tolist()}, expected {(counters + n).tolist()}")
        return torch.stack(out).cpu().numpy()


class CpuKernels:
    """CPU models of the kernels with their rounding points (fp32 arithmetic where the kernel has it), for running the
    checkers without a GPU.  ``fault`` plants one error."""

    def __init__(self, fault=None):
        self.fault = fault

    # SwiGLU
    def swiglu_fwd(self, gu, h):
        g, u = gu[:, 0::2], gu[:, 1::2]
        h.copy_(torch.nn.functional.silu(g) * u)

    def swiglu_bwd(self, gu, dh, dgu):
        g, u = gu[:, 0::2].double(), gu[:, 1::2].double()
        if self.fault == "swiglu_swap":
            g, u = u, g
        act, s = silu64(g)
        dact = rbf(dh.double() * u)
        dgu[:, 0::2] = rbf(dact * (s + g * s * (1 - s))).to(torch.bfloat16)
        dgu[:, 1::2] = rbf(dh.double() * rbf(act)).to(torch.bfloat16)

    # RMSNorm
    def rmsnorm_fwd(self, x, w, eps, out=None, rstd=None):
        H = x.shape[-1]
        if H > 8192 or H % 8:
            raise RuntimeError(f"tl_rmsnorm_fwd: H={H} must be a multiple of 8 and <= 8192")
        xf = x.float()
        r = 1.0 / torch.sqrt((xf * xf).sum(-1, keepdim=True) / H + eps)
        out.copy_((w.float() * (xf * r).to(torch.bfloat16).float()).to(torch.bfloat16))
        if rstd is not None:
            rstd.copy_(r.reshape(-1))

    def rope_table(self, inv_freq, max_pos):
        ang = torch.arange(max_pos, dtype=torch.float32)[:, None] * inv_freq[None, :]
        return torch.cos(ang).to(torch.bfloat16), torch.sin(ang).to(torch.bfloat16)

    def rope_kv_fwd(self, qkv, q_out, k_cache, v_cache, pos0_dev, cos, sin, qn, kn, eps, S, n_h, n_kv, d, kv_start=None):
        n_tok = qkv.shape[0]
        B, heads, half = n_tok // S, n_h + 2 * n_kv, d // 2
        pos0 = int(pos0_dev[0])
        x = qkv.view(B, S, heads, d).double()
        pos = pos0 + torch.arange(S)
        ks = kv_start.long() if kv_start is not None else torch.zeros(B, dtype=torch.long)
        rpos = (pos[None, :] - ks[:B, None]).clamp_min(0)
        cc, ss = cos.double()[rpos][:, :, None], sin.double()[rpos][:, :, None]
        qk = x[:, :, :n_h + n_kv]
        if qn is not None:
            w = torch.cat([qn.double().expand(n_h, d), kn.double().expand(n_kv, d)])
            r = f32(1.0 / torch.sqrt(f32((f32(qk) ** 2).sum(-1, keepdim=True) / d + float(np.float32(eps)))))
            qk = rbf(w * rbf(f32(qk * r)))
        o = rope_fwd_ref(qk, cc, ss).to(torch.bfloat16)
        q_out.view(B, S, n_h, d).copy_(o[:, :, :n_h])
        k_cache[:, :, pos0:pos0 + S] = o[:, :, n_h:].permute(0, 2, 1, 3)
        v_cache[:, :, pos0:pos0 + S] = qkv.view(B, S, heads, d)[:, :, n_h + n_kv:].permute(0, 2, 1, 3)

    def rope_kv_bwd(self, dq, dk, dv, dqkv, cos, sin, S, n_h, n_kv, d):
        n_tok, half, n_rep = dqkv.shape[0], d // 2, n_h // n_kv
        B = n_tok // S
        reps = n_rep - 1 if self.fault == "rope_nrep_minus_1" and n_rep > 1 else n_rep

        def part(t):   # fp32 sum of the partials in order
            v = t.float()[:, :, :S].view(B, n_kv, n_rep, S, d)
            acc = v[:, :, 0].clone()
            for r in range(1, reps):
                acc = acc + v[:, :, r]
            return acc.permute(0, 2, 1, 3).reshape(n_tok, n_kv, d).double()
        dqk = torch.cat([dq.double(), part(dk)], 1)
        pos = torch.arange(n_tok) % S
        if self.fault == "rope_pos_off_by_one":
            pos = (pos + 1).clamp_max(cos.shape[0] - 1)
        cc, ss = cos.double()[pos][:, None], sin.double()[pos][:, None]
        d1, d2 = dqk[..., :half], dqk[..., half:]
        o = torch.cat([torch.cat([rbf(f32(d1 * cc + d2 * ss)), rbf(f32(d2 * cc - d1 * ss))], -1), rbf(part(dv))], 1)
        dqkv.copy_(o.reshape(n_tok, -1).to(torch.bfloat16))

    def ce_fwd_bwd(self, logits, labels, loss_sum, n_valid, dlogits, scale):
        M, V = logits.shape
        x = logits.float()
        mx = x.max(-1, keepdim=True).values
        e = torch.exp(x - mx)
        se = e.sum(-1, keepdim=True)
        o = e * (np.float32(scale) / se)
        valid = (labels >= 0) & (labels < V)
        lab = labels.clamp(0, V - 1)
        if self.fault == "ce_label_off":
            lab = (lab + 1) % V
        rows = torch.arange(M)
        loss_sum += ((mx.squeeze(-1) + torch.log(se.squeeze(-1))) - x[rows, lab])[valid].sum()
        o[rows, lab] -= np.float32(scale)
        o[~valid] = 0
        dlogits.copy_(o.to(torch.bfloat16))

    def embed_fwd(self, ids, table, out):
        V = table.shape[0]
        out.copy_(table[torch.where((ids >= 0) & (ids < V), ids, torch.zeros_like(ids))])

    def add_inplace(self, a, b):
        a.copy_(rbf(f32(a.double() + b.double())).to(torch.bfloat16))

    def scale_add(self, a, b, scale, accumulate=True):
        s = float(np.float32(scale))
        acc = accumulate or self.fault == "scale_add_ignores_acc"
        v = f32(s * b.double() + (a.double() if acc else 0.0))
        a.copy_(rbf(v).to(torch.bfloat16) if a.dtype == torch.bfloat16 else v.float())

    def f32_to_bf16_accum(self, src, dst, accumulate):
        v = f32(src.double() + (dst.double() if accumulate else 0.0)).float()
        if self.fault == "f32_to_bf16_trunc":
            dst.copy_((v.view(torch.int32) & ~0xFFFF).view(torch.float32).to(torch.bfloat16))
        else:
            dst.copy_(v.to(torch.bfloat16))

    def adamw_step(self, p, g, m, v, lr, b1, b2, eps, wd, step, decoupled):
        n = p.numel()
        k = n - n % 8 if self.fault == "adam_no_tail" else n
        F = np.float32
        lr, b1, b2, eps, wd = F(lr), F(b1), F(b2), F(eps), F(wd)
        bc1, bc2s = (F(x) for x in host_bias_corrections(b1, b2, step))
        pw, gr, mi, vi = p[:k].float(), g[:k].float(), m[:k].clone(), v[:k].clone()
        if wd != 0:
            if decoupled:
                pw = pw * (F(1) - lr * wd)
            else:
                gr = gr + wd * pw
        mi = b1 * mi + (F(1) - b1) * gr
        vi = b2 * vi + (F(1) - b2) * gr * gr
        pw = pw - (lr / bc1) * (mi / (torch.sqrt(vi) / F(bc2s) + eps))
        m[:k], v[:k], p[:k] = mi, vi, pw.to(torch.bfloat16)

    def sample_many(self, c: SampleCase, logits, counters, prompt, eos, n):
        models = case_models(c, logits, prompt, eos, fault=self.fault)
        out = np.zeros((n, c.M), np.int64)
        for m, rm in enumerate(models):
            u = philox_u(SEED, m, np.arange(n, dtype=np.uint64) + int(counters[m]))
            out[:, m] = model_draws(rm, u, self.fault)[0]
        return out
