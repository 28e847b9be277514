"""Element-by-element checks of the Linear kernels (``tl_gemm_bf16``, ``tl_gemm_bf16_ws[_norm]``, ``tl_gemv_bf16[_pf]``).

Two legs, one harness:

  * exact: A and B are bf16 integers in [-4, 4]; bias, residual and the old C are small integers or exact halves.  Every
    product and every fp32 partial sum is then an integer below 2^24, so fp32 accumulation is exact in any order, whatever
    the tiling, the split or the K-block schedule, and the output follows bit for bit from the header's epilogue chain with
    the kernel's rounding points (``chain_exact``).  Only SwiGLU's silu is inexact: one bf16 ulp of silu times |up|, plus
    one ulp of the output.
  * rounding: bf16 normal inputs at the model's magnitudes.  Per element, |got - ref| <= one bf16 ulp per rounding point of
    the chain (carried through the later operations) + 2^-17 * sum_k |a_k b_k| for fp32 accumulation, ref being the
    unrounded chain in float64 (``chain_bound``).

Every operand and output sits in a guard buffer (``Guard``): pad rows before and after, and for GEMM a row pitch wider than
the logical width.  Operand pads hold NaN (a read past the logical extent poisons an exact result), output pads and the
bytes past the split-K workspace a sentinel bit pattern.  After a call every input buffer is unchanged bit for bit and
only C's logical region may differ from what it held.

``gemm_path`` / ``gemv_path`` restate the host dispatch (tile width, split count, GEMV ring, fallback) from the device's SM
count, so that each case can be checked to run the kernels it was written for.  ``path_matrix`` puts cases on both sides
of every threshold; ``model_calls`` lists every Linear call of ml/shard.py, ml/train.py and ml/stage.py for a config.

Nothing here needs a GPU: tests/test_linear_cases_cpu.py runs the checkers on a CPU model of the tiled GEMM.
"""
from __future__ import annotations

import hashlib
import json
import os
import re
import tempfile
from dataclasses import dataclass
from typing import Dict, List, Optional

import torch

EPI_BIAS, EPI_RESIDUAL, EPI_SWIGLU, EPI_OUT_F32, EPI_ACCUM, A_MN, B_MN = 1, 2, 4, 8, 16, 32, 64
BM, BK = 128, 64
EXACT_LIMIT = 2 ** 24           # fp32 integers are exact below this
ACC_REL = 2.0 ** -17            # fp32 accumulation term of the rounding bound, times sum |a b|
NORM_TIE_REL = 2.0 ** -16       # x * rstd this close (relative) to a bf16 rounding tie may round either way: the kernels'
                                # fp32 sum of squares over K <= 18,944 (<= 74 terms per thread, then a tree) is within
                                # about 2^-17.6 of the float64 one, and rstd within half of that
EPS = 1e-6
BF16_SENTINEL = 0x7FA5          # a NaN payload no kernel produces
F32_SENTINEL = 0x7FBADBAD
PAD_ROWS = 3
EXACT_MAX_ABS = 4               # |A|, |B| on the exact leg
EXACT_SMALL = 8                 # |bias|, |residual|, |C0| on the exact leg (multiples of 1/2)

_INT = {torch.bfloat16: torch.int16, torch.float32: torch.int32}


# ------------------------------------------------------------------------------------------------ cases
@dataclass(frozen=True)
class Case:
    name: str
    op: str                     # "gemm" | "gemv"
    M: int
    N: int
    K: int
    flags: int = 0              # EPI_* and *_MN bits
    alias: bool = False         # residual is C itself (out=x, residual=x)
    ws_bytes: int = 0           # split-K workspace handed to tl_gemm_bf16_ws[_norm] (0: tl_gemm_bf16)
    norm: bool = False          # GEMM: fused RMSNorm of C into H; GEMV: RMSNorm prologue of x
    ld_pad: int = 8             # GEMM: extra elements in every row pitch (a multiple of 8, as TMA requires)
    next_w: bool = False        # GEMV: tl_gemv_bf16_pf with an L2 prefetch of another weight

    @property
    def swiglu(self):
        return bool(self.flags & EPI_SWIGLU)

    @property
    def f32(self):
        return bool(self.flags & EPI_OUT_F32)

    @property
    def exact_ok(self):
        """the exact leg needs integer operands all the way: the GEMV norm prologue has none"""
        return not (self.op == "gemv" and self.norm)

    @property
    def c_cols(self):
        return self.N // 2 if self.swiglu else self.N

    def headroom(self) -> int:
        """largest |value| an fp32 partial sum or epilogue add can reach on the exact leg"""
        return self.K * EXACT_MAX_ABS ** 2 + 3 * EXACT_SMALL


def splitk_ws(M, N):
    """tl_gemm_splitk_ws"""
    return 8 * (0 if M > 128 else M) * N * 4


# ------------------------------------------------------------------------------------------------ dispatch restated
def split_plan(c: Case, sms: int):
    """(splits, kb_per) of tl_gemm_bf16_ws_norm's split-K branch, or None when it takes the plain path."""
    if c.op != "gemm" or not c.ws_bytes or c.flags & (A_MN | B_MN):
        return None
    tiles_n, num_k = -(-c.N // 128), -(-c.K // BK)
    if not (0 < c.M <= BM and c.K % 8 == 0 and c.N % 8 == 0 and tiles_n * 2 <= sms and num_k >= 16):
        return None
    splits = min(sms // tiles_n, 8)
    kb_per = max(8, -(-num_k // splits))
    splits = -(-num_k // kb_per)
    if splits > 1 and c.ws_bytes >= splits * c.M * c.N * 4:
        return splits, kb_per
    return None


def gemm_tile(c: Case, sms: int) -> int:
    b_mn = bool(c.flags & B_MN)
    return 32 if (c.M <= BM and not b_mn and -(-c.N // 128) < 2 * sms and c.N % 32 == 0) else 128


def gemm_path(c: Case, sms: int) -> dict:
    """kernels (in launch order, with grid.x) that one call of this case runs"""
    sp = split_plan(c, sms)
    a_mn, b_mn = str(bool(c.flags & A_MN)).lower(), str(bool(c.flags & B_MN)).lower()
    if sp:
        splits, kb_per = sp
        tiles = -(-c.M // BM) * -(-c.N // 128) * splits
        ks = [(f"gemm_bf16_kernel<128, false, false>", min(tiles, sms))]
        if c.norm:
            ks.append(("splitk_reduce_norm_kernel", c.M))
        else:
            ks.append(("splitk_reduce_kernel", -(-(c.M * (c.N // 8)) // 256)))
        return {"tile": 128, "splits": splits, "kb_per": kb_per, "kernels": ks}
    bn = gemm_tile(c, sms)
    tiles = -(-c.M // BM) * -(-c.N // bn)
    ks = [(f"gemm_bf16_kernel<{bn}, {a_mn}, {b_mn}>", min(tiles, sms))]
    if c.norm:
        ks.append(("rmsnorm_fwd_kernel", c.M))
    return {"tile": bn, "splits": 1, "kb_per": -(-c.K // BK), "kernels": ks}


def gemv_reg_params(m, N, K, sms):
    """(G, WPI, grid) of the register-streaming gemv_kernel"""
    nvec = K // 8
    wpi = 1
    while wpi < 8 and -(-nvec // (32 * wpi)) > 4:
        wpi *= 2
    slots = 8 // wpi
    npairs = N // 2
    g, wave = 4, sms * 2 * slots
    while g > 1 and npairs // g < 4 * wave:
        g //= 2
    iters = -(-nvec // (32 * wpi))
    if iters <= 4 and g < 2 and npairs >= 2 * wave:
        g = 2
    smem = m * K * 2 + 8 * 2 * g * m * 4
    per_sm = 1 if smem > 100 * 1024 else (2 if smem > 64 * 1024 else 4)
    grid = min(-(-(-(-npairs // g)) // slots), sms * per_sm)
    return g, wpi, grid


def gemv_stream_params(m, N, K, sms, env):
    """(per_sm, P, chunked, grid) of gemv_stream_kernel<m>, or None when fewer than 4 ring stages fit (fallback)"""
    forced = env.get("TL_GEMV_CTAS_PER_SM", "")
    forced = 2 if forced[:1] == "2" else (1 if forced[:1] == "1" else 0)
    per_sm = forced or (2 if (N * K * 2) // sms <= 128 * 1024 else 1)
    ring_kb = int(env.get("TL_GEMV_RING_KB", "220") or 220)
    if ring_kb < 48 or ring_kb > 220:
        ring_kb = 220
    cap = 110 * 1024 if per_sm == 2 else ring_kb * 1024
    fixed = ((m * K * 2 + 15) & ~15) + 2 * 16 * 8
    chunked = K > 4096 or K * 4 > 16384
    P = 1 if chunked else max(1, min(8, 16384 // (K * 4)))
    stage = 16384 if chunked else (P * K * 4 + 127) & ~127
    if min(16, (cap - fixed) // stage) < 4:
        return None
    return per_sm, P, chunked, min(sms * per_sm, N // 2)


def gemv_mma_applies(c: Case, env):
    if env.get("TL_GEMV_MMA", "")[:1] != "1" or env.get("TL_GEMV_IMPL", "")[:1] == "r":
        return None
    if c.M < 2 or c.N % 16 or c.K % 16:
        return None
    x_in_stage = 8 * (2 * c.K + 16) + 256 + 6 * 16640 > 220 * 1024
    if x_in_stage and c.norm:
        return None
    return {"x_in_stage": x_in_stage}


def gemv_path(c: Case, sms: int, env: Optional[Dict[str, str]] = None) -> dict:
    env = dict(os.environ) if env is None else env
    mma = gemv_mma_applies(c, env)
    if mma is not None:
        return {"kernels": [("gemv_mma_kernel", min(sms, c.N >> 4))], "mma": mma}
    stream_ok = env.get("TL_GEMV_IMPL", "")[:1] != "r"
    ks, kinds = [], []
    done = 0
    while done < c.M:
        m = min(4, c.M - done)
        sp = gemv_stream_params(m, c.N, c.K, sms, env) if stream_ok else None
        if sp:
            ks.append((f"gemv_stream_kernel<{m}>", sp[3]))
            kinds.append({"m": m, "per_sm": sp[0], "P": sp[1], "chunked": sp[2]})
        else:
            g, wpi, grid = gemv_reg_params(m, c.N, c.K, sms)
            ks.append((f"gemv_kernel<{m}, {g}, {wpi}>", grid))
            kinds.append({"m": m, "g": g, "wpi": wpi})
        done += m
    return {"kernels": ks, "chunks": kinds}


def path_of(c: Case, sms: int, env=None) -> dict:
    return gemm_path(c, sms) if c.op == "gemm" else gemv_path(c, sms, env)


# ------------------------------------------------------------------------------------------------ guard buffers
class Guard:
    """A rows x cols matrix with row pitch ld inside a buffer of pad rows before and after (its first element 16-byte
    aligned).  Everything outside the matrix holds ``fill_bits``; ``outside_changed`` lists where it no longer does."""

    def __init__(self, rows, cols, ld, dtype, device, fill_bits, pad=PAD_ROWS):
        assert ld >= cols, (cols, ld)
        al = 16 // torch.empty(0, dtype=dtype).element_size()
        self.rows, self.cols, self.ld, self.pad, self.dtype = rows, cols, ld, pad, dtype
        self.fill_bits = fill_bits
        self.start = (pad * ld + al - 1) // al * al
        self.buf = torch.empty(self.start + (rows + pad) * ld, dtype=dtype, device=device)
        self.bits = self.buf.view(_INT[dtype])
        self.bits.fill_(fill_bits)
        self.rows_view = self.buf[self.start:self.start + rows * ld].view(rows, ld)     # the matrix and its pitch slack
        self.t = self.rows_view[:, :cols]

    @property
    def ptr(self):
        return self.t.data_ptr()

    def snapshot(self):
        return self.bits.clone()

    def outside_changed(self):
        """(row, col) of changed guard elements, rows relative to the matrix's first row (negative: before it)"""
        bad = self.bits != self.fill_bits
        bad[self.start:self.start + self.rows * self.ld].view(self.rows, self.ld)[:, :self.cols] = False
        idx = bad.nonzero()[:, 0] - self.start
        return torch.stack([torch.div(idx, self.ld, rounding_mode="floor"), torch.remainder(idx, self.ld)], 1)


def nan_bits(dtype):
    return 0x7FC0 if dtype == torch.bfloat16 else 0x7FC00000


def sentinel_bits(dtype):
    return BF16_SENTINEL if dtype == torch.bfloat16 else F32_SENTINEL


def vec_guard(n, device, dtype=torch.bfloat16):
    """a 1-D operand (bias, norm gain) with NaN on both sides"""
    return Guard(1, n, (n + 7) // 8 * 8, dtype, device, nan_bits(dtype), pad=1)


# ------------------------------------------------------------------------------------------------ operands
def _gen(seed, device):
    g = torch.Generator(device=device)
    g.manual_seed(seed & 0x7FFFFFFF)
    return g


def _seed(name, tag):
    return int.from_bytes(hashlib.sha256(f"{name}/{tag}".encode()).digest()[:4], "little")


def _ints(shape, lim, seed, device, halves=False):
    g = _gen(seed, device)
    if halves:
        return torch.randint(-2 * lim, 2 * lim + 1, shape, generator=g, device=device).float() / 2
    return torch.randint(-lim, lim + 1, shape, generator=g, device=device).float()


def _normal(shape, std, seed, device):
    g = _gen(seed, device)
    return torch.randn(shape, generator=g, device=device) * std


def make_buffers(c: Case, leg: str, device) -> dict:
    """Guarded operands and outputs of one call, filled for the leg ("exact" | "round")."""
    bf = torch.bfloat16
    exact = leg == "exact"
    pad = c.ld_pad if c.op == "gemm" else 0
    out_dtype = torch.float32 if c.f32 else bf
    b = {}

    def fill(name, shape, std, lim, halves=False):
        return (_ints(shape, lim, _seed(c.name, name), device, halves) if exact
                else _normal(shape, std, _seed(c.name, name), device))

    if c.op == "gemm":
        a_rows, a_cols = (c.K, c.M) if c.flags & A_MN else (c.M, c.K)
        b_rows, b_cols = (c.K, c.N) if c.flags & B_MN else (c.N, c.K)
        b["a"] = Guard(a_rows, a_cols, a_cols + pad, bf, device, nan_bits(bf))
        b["b"] = Guard(b_rows, b_cols, b_cols + pad, bf, device, nan_bits(bf))
        b["a"].t.copy_(fill("a", (a_rows, a_cols), 1.0, EXACT_MAX_ABS))
        b["b"].t.copy_(fill("b", (b_rows, b_cols), 0.05, EXACT_MAX_ABS))
        ldc = c.c_cols + (0 if c.norm else pad)
    else:
        b["a"] = Guard(c.M, c.K, c.K, bf, device, nan_bits(bf))
        b["b"] = Guard(c.N, c.K, c.K, bf, device, nan_bits(bf))
        b["a"].t.copy_(fill("a", (c.M, c.K), 2.0 if c.norm else 1.0, EXACT_MAX_ABS))
        b["b"].t.copy_(fill("b", (c.N, c.K), 0.05, EXACT_MAX_ABS))
        ldc = c.c_cols
    b["c"] = Guard(c.M, c.c_cols, ldc, out_dtype, device, sentinel_bits(out_dtype))
    if c.flags & EPI_ACCUM:
        b["c"].t.copy_(fill("c0", (c.M, c.c_cols), 0.5, EXACT_SMALL, halves=True))
    if c.flags & EPI_BIAS:
        b["bias"] = vec_guard(c.N, device)
        b["bias"].t.copy_(fill("bias", (1, c.N), 0.5, EXACT_SMALL, halves=True))
    if c.flags & EPI_RESIDUAL:
        r = fill("res", (c.M, c.N), 1.0, EXACT_SMALL, halves=True)
        if c.alias:
            b["c"].t.copy_(r)
        else:       # the GEMM reads the residual with C's pitch (ldr = ldc), the GEMV with pitch N
            b["res"] = Guard(c.M, c.N, ldc if c.op == "gemm" else c.N, bf, device, nan_bits(bf))
            b["res"].t.copy_(r)
    if c.norm:
        b["g"] = vec_guard(c.N if c.op == "gemm" else c.K, device)
        b["g"].t.copy_((1 + 0.1 * _normal((1, b["g"].cols), 1.0, _seed(c.name, "g"), device)))
        if c.op == "gemm":
            b["h"] = Guard(c.M, c.N, c.N, bf, device, BF16_SENTINEL)
    if c.ws_bytes:
        n = c.ws_bytes // 4
        b["ws"] = Guard(1, n, (n + 3) // 4 * 4 + 64, torch.float32, device, F32_SENTINEL, pad=0)   # 256 B past its end
    if c.next_w:
        b["next"] = Guard(1024, 4096, 4096, bf, device, nan_bits(bf), pad=0)
        b["next"].t.copy_(_normal((1024, 4096), 0.05, 7, device))
    return b


def input_names(c: Case, bufs):
    return [k for k in bufs if k not in ("c", "h", "ws")]


# ------------------------------------------------------------------------------------------------ references
def rbf(x):
    """float64 -> the value a bf16 tensor would hold (fp32 then RNE to bf16, as the kernels round fp32 values)"""
    return x.to(torch.float32).to(torch.bfloat16).to(torch.float64)


def r32(x):
    return x.to(torch.float32).to(torch.float64)


def ulp_bf16(x):
    _, e = torch.frexp(x.abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(x), (e - 8).to(torch.int32))


def ulp_f32(x):
    _, e = torch.frexp(x.abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(x), (e - 24).to(torch.int32))


def silu64(x):
    return x / (1 + torch.exp(-x))


def silu_slack(g, s):
    """how far the kernels' bf16 silu(g) may lie from the float64 one: one bf16 ulp, and all of it below g = -87, where
    fp32 exp(-g) overflows and x / (1 + exp(-x)) flushes to zero"""
    return ulp_bf16(s.abs() * (1 + 2.0 ** -7)) + (g < -87) * s.abs()


def norm_prologue(x, g):
    """h = bf16(g * bf16(x * rstd)) with a float64 rstd; near[m,k] marks x*rstd within NORM_TIE_REL of a rounding tie,
    slack[m,k] the most h can move there (one ulp of the normalised value times |g|, plus one ulp of h)"""
    rstd = 1.0 / torch.sqrt((x * x).mean(-1, keepdim=True) + EPS)
    t = x * rstd
    n = rbf(t)
    h = rbf(g * n)
    u = ulp_bf16(t)
    frac = torch.remainder(t.abs() / u, 1.0)
    near = (frac - 0.5).abs() <= NORM_TIE_REL * t.abs() / u
    slack = near * (g.abs() * ulp_bf16(n) * 1.01 + ulp_bf16(h))
    return h, slack


def chain_exact(c: Case, acc, bias, res, old):
    """(want, tol): the output the header's chain gives, rounded where the kernel rounds; tol is 0 except for SwiGLU"""
    v = r32(acc + bias) if bias is not None else acc
    if c.swiglu:
        g, u = rbf(v[:, 0::2]), rbf(v[:, 1::2])
        s = silu64(g)
        want = rbf(rbf(s) * u)
        return want, silu_slack(g, s) * u.abs() + ulp_bf16(want)
    if c.f32:
        want = r32(v + old) if old is not None else r32(v)
        return want, torch.zeros_like(want)
    t = rbf(v)
    if res is not None:
        t = r32(t + res)
    if old is not None:
        t = r32(t + old)
    want = rbf(t)
    return want, torch.zeros_like(want)


def chain_bound(c: Case, acc, absacc, extra, bias, res, old):
    """(ref, bound): the unrounded chain in float64 and the per-element bound"""
    E = ACC_REL * absacc
    if extra is not None:
        E = E + extra
    v = acc + bias if bias is not None else acc
    if bias is not None:
        E = E + ulp_f32(v)
    if c.swiglu:
        g, u, Eg, Eu = v[:, 0::2], v[:, 1::2], E[:, 0::2], E[:, 1::2]
        eg = Eg + ulp_bf16(g.abs() + Eg)
        eu = Eu + ulp_bf16(u.abs() + Eu)
        s = silu64(g)
        es = 1.1 * eg + silu_slack(g, s) + 2.0 ** -20 * s.abs()
        ref = s * u
        b1 = (s.abs() + es) * eu + u.abs() * es
        return ref, b1 + ulp_bf16(ref.abs() + b1)
    if c.f32:
        ref = v + old if old is not None else v
        return ref, E + ulp_f32(v.abs() + E) + (ulp_f32(ref.abs() + E) if old is not None else 0)
    bound = E + ulp_bf16(v.abs() + E)
    ref = v
    if res is not None:
        ref = ref + res
    if old is not None:
        ref = ref + old
    if res is not None or old is not None:
        bound = bound + ulp_bf16(ref.abs() + bound)
    return ref, bound


def norm_check(C, H, g):
    """H = g * bf16(C * rstd(C)) for the bf16 C the call wrote: bit-exact except where C*rstd is near a rounding tie
    (the kernels' fp32 rstd may round it the other way), and there within the flip's slack"""
    want, slack = norm_prologue(C.double(), g.double())
    d = (H.double() - want).abs()
    return (d > slack) | torch.isnan(H.double()), want


# ------------------------------------------------------------------------------------------------ failure reports
def describe(c: Case, path: dict, blocks, what: str, limit=8) -> str:
    """the mismatching (row, column) coordinates, grouped by 128 x BN output tile and naming the split plan;
    blocks = [(first row, bad coordinates in the block, got, want, count)]"""
    n = sum(b[4] for b in blocks)
    idx = torch.cat([b[1] + torch.tensor([b[0], 0], device=b[1].device) for b in blocks]).cpu()
    bn = path.get("tile", 0) if c.op == "gemm" else 0
    msg = [f"{c.name}: {what}: {n} of {c.M * c.c_cols} elements wrong (M={c.M} N={c.N} K={c.K} flags={c.flags:#x}"
           f" kernels={path.get('kernels')} splits={path.get('splits', 1)} kb_per={path.get('kb_per', '-')})"]
    if bn:
        col_n = idx[:, 1] * (2 if c.swiglu else 1)           # column in the N space of B's rows
        tiles: Dict[tuple, int] = {}
        for r, cn in zip((idx[:, 0] // BM).tolist(), (col_n // bn).tolist()):
            tiles[(r, cn)] = tiles.get((r, cn), 0) + 1
        top = sorted(tiles.items(), key=lambda kv: -kv[1])[:limit]
        msg.append(f"  by 128x{bn} tile (tile_m, tile_n), first {idx.shape[0]} coordinates: "
                   + ", ".join(f"{k}: {v}" for k, v in top) + (f" ... ({len(tiles)} tiles)" if len(tiles) > limit else ""))
    shown = 0
    for r0, bidx, got, want, _ in blocks:
        for r, col in bidx[:limit - shown].tolist():
            msg.append(f"  ({r0 + r}, {col}): got {got[r, col].item()!r} want {want[r, col].item()!r}")
            shown += 1
    return "\n".join(msg)


def describe_guard(name, idx, limit=8):
    if idx.shape[0] == 0:
        return ""
    return f"{name}: {idx.shape[0]} guard elements changed, first at (row, col) " + \
        ", ".join(str(tuple(x)) for x in idx[:limit].tolist())


# ------------------------------------------------------------------------------------------------ one call, checked
def check_call(c: Case, leg: str, launch, device, sms: int = 132, env=None, want_bits=False) -> dict:
    """Build the guarded buffers of ``c``, call ``launch(c, bufs)``, check the leg's criterion and the guards.
    Returns {"errors": [...], "ratio": worst |err| / bound (rounding leg), "bits": sha-256 of C (and H) if asked}.
    The float64 reference is computed in blocks of rows, so that vocabulary-sized outputs fit beside their operands."""
    assert leg in ("exact", "round") and (leg == "round" or c.exact_ok), (c.name, leg)
    bufs = make_buffers(c, leg, device)
    path = path_of(c, sms, env)
    snaps = {k: bufs[k].snapshot() for k in input_names(c, bufs)}
    c0 = bufs["c"].t.clone()
    launch(c, bufs)
    errs = []
    for k in snaps:
        ch = (bufs[k].bits != snaps[k]).nonzero()
        if ch.numel():
            errs.append(f"{c.name}: input {k} changed at {ch.shape[0]} elements, first flat index {ch[0].item()}")
    del snaps
    for k, what in (("c", "output C"), ("h", "output H"), ("ws", "bytes past the workspace")):
        if k in bufs:
            e = describe_guard(f"{c.name}: {what}", bufs[k].outside_changed())
            if e:
                errs.append(e)
    if leg == "exact":
        assert c.headroom() < EXACT_LIMIT, c
    b = bufs["b"].t.double()
    if c.flags & B_MN:
        b = b.t()
    babs = b.abs()
    g = bufs["g"].t.double() if (c.norm and c.op == "gemv") else None
    bias = bufs["bias"].t.double()[0] if "bias" in bufs else None
    rb = max(1, (1 << 26) // max(c.N, c.K))
    ratio = 0.0
    bad_all, got_all, want_all = [], [], []
    for r0 in range(0, c.M, rb):
        r1 = min(c.M, r0 + rb)
        a = bufs["a"].t[:, r0:r1].double().t() if c.flags & A_MN else bufs["a"].t[r0:r1].double()
        extra = None
        if g is not None:
            a, slack = norm_prologue(a, g)
            extra = slack @ babs.t()
        acc = a @ b.t()
        old_blk = c0[r0:r1].double()
        res = None
        if c.flags & EPI_RESIDUAL:
            res = old_blk if c.alias else bufs["res"].t[r0:r1].double()
        old = old_blk if c.flags & EPI_ACCUM else None
        got = bufs["c"].t[r0:r1].double()
        if leg == "exact":
            want, tol = chain_exact(c, acc, bias, res, old)
            bad = ((got - want).abs() > tol) | torch.isnan(got)
        else:
            absacc = a.abs() @ babs.t()
            want, bound = chain_bound(c, acc, absacc, extra, bias, res, old)
            err = (got - want).abs()
            bad = (err > bound) | torch.isnan(got)
            if not bool(torch.isnan(got).any()):
                ratio = max(ratio, float((err / bound).max()))
        if bool(bad.any()):
            bad_all.append((r0, bad.nonzero()[:64], got, want, int(bad.sum())))
    if bad_all:
        errs.append(describe(c, path, bad_all, "exact leg" if leg == "exact" else "rounding leg (|got - ref| > bound)"))
    if c.op == "gemm" and c.norm:
        hbad, hwant = norm_check(bufs["c"].t, bufs["h"].t, bufs["g"].t[0])
        if bool(hbad.any()):
            errs.append(describe(c, path, [(0, hbad.nonzero()[:64], bufs["h"].t.double(), hwant, int(hbad.sum()))],
                                 "fused RMSNorm output H"))
    out = {"errors": errs, "ratio": ratio, "path": path}
    if want_bits:
        for k in ("c", "h"):
            if k in bufs:
                t = bufs[k].t.contiguous().view(_INT[bufs[k].dtype]).cpu().numpy().tobytes()
                out["bits_" + k] = hashlib.sha256(t).hexdigest()
    return out


# ------------------------------------------------------------------------------------------------ the native calls
def native_launch(nat, prefetch_bytes=8 << 20):
    """launch(c, bufs) through the C ABI with explicit pitches (the Python wrappers take contiguous tensors only)"""
    lib = nat.load()

    def ptr(bufs, k):
        return bufs[k].ptr if k in bufs else None

    def launch(c: Case, bufs):
        st = nat._stream()
        a, b, C = bufs["a"], bufs["b"], bufs["c"]
        res = C.ptr if c.alias else ptr(bufs, "res")
        if c.op == "gemm":
            ws = ptr(bufs, "ws")
            if c.norm:
                rc = lib.tl_gemm_bf16_ws_norm(a.ptr, b.ptr, C.ptr, c.M, c.N, c.K, a.ld, b.ld, C.ld, ptr(bufs, "bias"), res,
                                              c.flags, ws, c.ws_bytes, bufs["g"].ptr, EPS, bufs["h"].ptr, st)
            elif c.ws_bytes:
                rc = lib.tl_gemm_bf16_ws(a.ptr, b.ptr, C.ptr, c.M, c.N, c.K, a.ld, b.ld, C.ld, ptr(bufs, "bias"), res,
                                         c.flags, ws, c.ws_bytes, st)
            else:
                rc = lib.tl_gemm_bf16(a.ptr, b.ptr, C.ptr, c.M, c.N, c.K, a.ld, b.ld, C.ld, ptr(bufs, "bias"), res,
                                      c.flags, st)
        elif c.next_w:
            rc = lib.tl_gemv_bf16_pf(a.ptr, b.ptr, C.ptr, c.M, c.N, c.K, ptr(bufs, "bias"), res, ptr(bufs, "g"), EPS,
                                     c.flags, bufs["next"].ptr, prefetch_bytes, st)
        else:
            rc = lib.tl_gemv_bf16(a.ptr, b.ptr, C.ptr, c.M, c.N, c.K, ptr(bufs, "bias"), res, ptr(bufs, "g"), EPS,
                                  c.flags, st)
        nat._check(rc, c.name)
    return launch


class KernelLog:
    """Names and grid sizes of the project's kernels launched inside the block, from torch.profiler (CUPTI activity
    tracing of this process)."""

    def __enter__(self):
        self.prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA])
        self.prof.__enter__()
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        self.prof.__exit__(*exc)
        with tempfile.TemporaryDirectory() as d:
            p = os.path.join(d, "trace.json")
            self.prof.export_chrome_trace(p)
            with open(p) as f:
                ev = json.load(f).get("traceEvents", [])
        ks = sorted((e for e in ev if e.get("cat") == "kernel"), key=lambda e: e.get("ts", 0))
        self.all_names = [e.get("name", "") for e in ks]
        self.kernels = []
        for e in ks:
            m = re.search(r"tl::([A-Za-z0-9_]+(?:<[^>()]*>)?)", e.get("name", ""))
            if m:
                self.kernels.append((m.group(1), (e.get("args", {}).get("grid") or [None])[0]))
        return False


def match_paths(expected: List[tuple], kernels: List[tuple], all_names: List[str]) -> str:
    """expected: [(case name, [(kernel, grid), ...])] in call order; '' when the recorded kernels match exactly"""
    if not all_names:
        return "torch.profiler recorded no CUDA kernels: the path of no case is proven"
    if not kernels:
        return f"torch.profiler recorded {len(all_names)} kernels but none of tl::, first: {all_names[:3]}"
    i = 0
    for name, ks in expected:
        got = kernels[i:i + len(ks)]
        if [k for k, _ in got] != [k for k, _ in ks] or [g for _, g in got] != [g for _, g in ks]:
            return f"{name}: expected kernels (name, grid.x) {ks}, recorded {got}"
        i += len(ks)
    if i != len(kernels):
        return f"{len(kernels) - i} unexpected kernels after the last case: {kernels[i:i + 4]}"
    return ""


# ------------------------------------------------------------------------------------------------ CPU model (self-test)
FAULTS = ("drop_kblock", "oob_store", "nan_read", "stale_row", "truncate", "swap_gate_up", "plus2pct")


def cpu_gemm(fault: Optional[str] = None):
    """launch(c, bufs) for a CPU model of the tiled GEMM: fp32 sums per 64-wide K block, added block by block, the
    epilogue in fp32 with the kernel's bf16 rounding points.  ``fault`` plants one of FAULTS."""

    def launch(c: Case, bufs):
        A, B = bufs["a"], bufs["b"]
        a = A.t.float()
        if fault == "nan_read":         # one row reads one element past its last column (the NaN pitch pad)
            a = a.clone()
            a[0, -1] = A.rows_view[0, A.cols].float()
        b = B.t.float()
        if c.flags & A_MN:
            a = a.t()
        if c.flags & B_MN:
            b = b.t()
        M, N, K = c.M, c.N, c.K
        acc = torch.zeros(M, N, dtype=torch.float32)
        for k0 in range(0, K, BK):
            part = a[:, k0:k0 + BK] @ b[:, k0:k0 + BK].t()
            if fault == "drop_kblock" and k0 == BK:
                part[:BM, :32] = 0          # tile (0, 0) misses its second K block
            acc = acc + part
        v = acc
        if c.flags & EPI_BIAS:
            v = v + bufs["bias"].t[0].float()
        C = bufs["c"]
        if c.swiglu:
            g, u = v[:, 0::2].bfloat16().float(), v[:, 1::2].bfloat16().float()
            if fault == "swap_gate_up":
                g[:, 1], u[:, 1] = u[:, 1].clone(), g[:, 1].clone()
            out = ((g / (1 + torch.exp(-g))).bfloat16().float() * u)
        elif c.f32:
            out = v + C.t.float() if c.flags & EPI_ACCUM else v
        else:
            t = v.bfloat16().float()
            if c.flags & EPI_RESIDUAL:
                t = t + (C.t.float() if c.alias else bufs["res"].t.float())
            if c.flags & EPI_ACCUM:
                t = t + C.t.float()
            out = t
        if fault == "truncate" and not c.f32:
            col = out[:, 3].contiguous()
            out[:, 3] = (col.view(torch.int32) & ~0xFFFF).view(torch.float32)
        out = out.to(C.dtype)
        if fault == "plus2pct":
            r, col = divmod(int(out.float().abs().argmax()), out.shape[1])
            out[r, col] = (out[r, col].float() * 1.02).to(C.dtype)
        if fault == "stale_row":        # the last row of the ragged last row tile is never stored
            C.t[:M - 1].copy_(out[:M - 1])
        else:
            C.t.copy_(out)
        if fault == "oob_store":        # one 16-byte vector one column past N in row 0
            C.rows_view[0, C.cols:C.cols + 16 // C.buf.element_size()] = out[0, :16 // C.buf.element_size()]
        if c.norm:
            Cf = C.t.double()
            rstd = 1.0 / torch.sqrt((Cf * Cf).mean(-1, keepdim=True) + EPS)
            bufs["h"].t.copy_(rbf(bufs["g"].t.double() * rbf(Cf * rstd)))
    return launch


# ------------------------------------------------------------------------------------------------ case tables
GEMM_EPILOGUES = {
    "plain": dict(flags=0),
    "bias": dict(flags=EPI_BIAS),
    "res": dict(flags=EPI_RESIDUAL),
    "res_inplace": dict(flags=EPI_RESIDUAL, alias=True),
    "bias_res": dict(flags=EPI_BIAS | EPI_RESIDUAL),
    "swiglu": dict(flags=EPI_SWIGLU | EPI_BIAS),
    "f32": dict(flags=EPI_OUT_F32 | EPI_BIAS),
    "acc_bf16": dict(flags=EPI_ACCUM),
    "acc_f32": dict(flags=EPI_OUT_F32 | EPI_ACCUM),
}
MAJORS = {"kk": 0, "kB": B_MN, "Ak": A_MN, "AB": A_MN | B_MN}


def gemm_path_matrix(sms: int) -> List[Case]:
    """the 4 operand majors x every epilogue on 32- and 128-wide tiles with ragged M and N; short and ragged K; split-K
    at every split count, with and without the fused norm, on both sides of each SM-count threshold"""
    cs = []
    for mj, mf in MAJORS.items():
        for ep, kw in GEMM_EPILOGUES.items():
            for tile, (M, N) in (("t32", (72, 352)), ("t128", (200, 272))):
                if tile == "t32" and mf & B_MN:
                    continue            # B MN-major always takes 128-wide tiles
                ld_pad = {"kk": 8, "kB": 64, "Ak": 72, "AB": 8}[mj]
                c = Case(f"gemm.{mj}.{ep}.{tile}", "gemm", M, N, 136, flags=kw["flags"] | mf,
                         alias=kw.get("alias", False), ld_pad=ld_pad)
                cs.append(c)
    # K below 64, K % 64 != 0 with ragged M, K % 8 != 0 with both operands MN-major
    cs += [Case("gemm.k40.t32", "gemm", 24, 96, 40, flags=EPI_BIAS),
           Case("gemm.k40.t128", "gemm", 136, 136, 40, flags=EPI_RESIDUAL),
           Case("gemm.k8", "gemm", 8, 64, 8),
           Case("gemm.k200.ragged", "gemm", 129, 1032, 200, flags=EPI_BIAS | EPI_RESIDUAL, ld_pad=72),
           Case("gemm.AB.k52", "gemm", 136, 264, 52, flags=A_MN | B_MN | EPI_OUT_F32),
           Case("gemm.AB.k52.acc", "gemm", 136, 264, 52, flags=A_MN | B_MN | EPI_ACCUM),
           Case("gemm.AB.k2100", "gemm", 256, 136, 2100, flags=A_MN | B_MN | EPI_ACCUM, ld_pad=64)]
    # the 32-wide-tile threshold: ceil(N/128) < 2 * SMs, and M <= 128
    n32 = 256 * sms
    cs += [Case("gemm.t32.below", "gemm", 16, n32 - 128, 64, flags=EPI_BIAS),
           Case("gemm.t32.above", "gemm", 16, n32, 64, flags=EPI_BIAS),
           Case("gemm.m128", "gemm", 128, 352, 136),
           Case("gemm.m129", "gemm", 129, 352, 136)]
    # split-K: every split count the formula produces (tiles_n = 2 leaves min(8, SMs/2) splits)
    s0 = min(8, sms // 2)
    for s in range(2, s0 + 1):
        cs.append(Case(f"gemm.split{s}", "gemm", 33, 256, 512 * s, flags=EPI_BIAS | EPI_RESIDUAL, ws_bytes=splitk_ws(33, 256),
                       ld_pad=0))
    cs += [Case("gemm.split.lastblock", "gemm", 33, 256, 512 * 3 + 24, flags=EPI_BIAS, ws_bytes=splitk_ws(33, 256), ld_pad=0),
           Case("gemm.split.swiglu", "gemm", 17, 512, 4096, flags=EPI_SWIGLU | EPI_BIAS, ws_bytes=splitk_ws(17, 512), ld_pad=0),
           Case("gemm.split.f32", "gemm", 17, 256, 4096, flags=EPI_OUT_F32 | EPI_BIAS, ws_bytes=splitk_ws(17, 256), ld_pad=0),
           Case("gemm.split.f32acc", "gemm", 17, 256, 4096, flags=EPI_OUT_F32 | EPI_ACCUM, ws_bytes=splitk_ws(17, 256), ld_pad=0),
           Case("gemm.split.acc", "gemm", 17, 256, 4096, flags=EPI_ACCUM | EPI_RESIDUAL, ws_bytes=splitk_ws(17, 256), ld_pad=0),
           Case("gemm.split.inplace", "gemm", 64, 1024, 2048, flags=EPI_RESIDUAL, alias=True, ws_bytes=splitk_ws(64, 1024), ld_pad=0),
           Case("gemm.split.numk15", "gemm", 33, 256, 15 * 64, flags=EPI_BIAS, ws_bytes=splitk_ws(33, 256), ld_pad=0),
           Case("gemm.split.numk16", "gemm", 33, 256, 16 * 64, flags=EPI_BIAS, ws_bytes=splitk_ws(33, 256), ld_pad=0),
           Case("gemm.split.m129", "gemm", 129, 256, 2048, flags=EPI_BIAS, ws_bytes=splitk_ws(128, 256), ld_pad=0),
           Case("gemm.split.ws_short", "gemm", 33, 256, 2048, flags=EPI_BIAS,
                ws_bytes=4 * 33 * 256 * 4 - 16, ld_pad=0),
           Case("gemm.split.mn_major", "gemm", 32, 256, 2048, flags=B_MN, ws_bytes=splitk_ws(32, 256), ld_pad=0)]
    nt = sms // 2                           # tiles_n * 2 <= SMs: the widest N that still splits
    cs += [Case("gemm.split.tiles_at", "gemm", 8, 128 * nt, 2048, flags=EPI_RESIDUAL, ws_bytes=splitk_ws(8, 128 * nt), ld_pad=0),
           Case("gemm.split.tiles_over", "gemm", 8, 128 * (nt + 1), 2048, flags=EPI_RESIDUAL,
                ws_bytes=splitk_ws(8, 128 * (nt + 1)), ld_pad=0)]
    # the fused norm: split-K with the fused reduce, and the plain path followed by rmsnorm_fwd (N > 8192 is rejected)
    cs += [Case("gemm.norm.fused", "gemm", 5, 3584, 18944 // 4, flags=EPI_RESIDUAL, alias=True, ws_bytes=splitk_ws(5, 3584),
                norm=True, ld_pad=0),
           Case("gemm.norm.fused_bias", "gemm", 40, 896, 4864, flags=EPI_BIAS | EPI_RESIDUAL, ws_bytes=splitk_ws(40, 896),
                norm=True, ld_pad=0),
           Case("gemm.norm.plain", "gemm", 40, 896, 512, flags=EPI_RESIDUAL, alias=True, ws_bytes=splitk_ws(40, 896), norm=True,
                ld_pad=0)]
    return cs


GEMV_FORMS = {
    "plain": dict(flags=0),
    "bias": dict(flags=EPI_BIAS),
    "res_inplace": dict(flags=EPI_RESIDUAL, alias=True),
    "bias_res": dict(flags=EPI_BIAS | EPI_RESIDUAL),
    "swiglu": dict(flags=EPI_SWIGLU | EPI_BIAS),
    "norm_bias": dict(flags=EPI_BIAS, norm=True),
    "norm_swiglu": dict(flags=EPI_SWIGLU, norm=True),
}


def gemv_shapes(sms: int) -> dict:
    """GEMV shapes by the stream kernel's regime, from the SM count"""
    small_n = max(16, (128 * 1024 * sms) // (2 * 896) // 16 * 16)      # N*K*2/SMs <= 128 KB: two CTAs per SM
    return {
        "pairs2cta": (min(small_n, 2048), 896),       # whole pairs per stage (P = 4), two CTAs per SM
        "pairs1cta": ((128 * 1024 * sms // (2 * 896) // 16 + 64) * 16, 896),   # P = 4, one CTA per SM
        "chunked": (1024, 4864),                      # K > 4096: one 4096-column chunk of one pair per stage
        "chunked1cta": (4096, 4864),
        "chunked_odd": (130, 8200),                   # ragged last chunk, N not a multiple of 4
    }


def gemv_path_matrix(sms: int) -> List[Case]:
    cs = []
    for M in range(1, 9):
        for form, kw in GEMV_FORMS.items():
            for reg, (N, K) in gemv_shapes(sms).items():
                if M not in (1, 3, 4, 5, 8) and reg != "chunked":
                    continue
                cs.append(Case(f"gemv.m{M}.{form}.{reg}", "gemv", M, N, K, flags=kw["flags"], alias=kw.get("alias", False),
                               norm=kw.get("norm", False), ld_pad=0))
    # the register-streaming fallback, reached when fewer than 4 ring stages fit beside x
    cs += [Case("gemv.fallback.m3k8192", "gemv", 3, 1024, 8192, flags=EPI_BIAS, ld_pad=0),
           Case("gemv.fallback.m8k8192", "gemv", 8, 1024, 8192, flags=EPI_RESIDUAL, alias=True, ld_pad=0),
           Case("gemv.fallback.m4k20480", "gemv", 4, 4096, 20480, flags=EPI_SWIGLU, norm=True, ld_pad=0)]
    return cs


def gemv_mma_cases() -> List[Case]:
    """TL_GEMV_MMA=1: resident x (K = 896) and x streamed with the weights (K = 8192, no norm prologue)"""
    cs = []
    for M in (2, 5, 8):
        cs += [Case(f"gemv.mma.m{M}.resident", "gemv", M, 1152, 896, flags=EPI_BIAS, norm=True, ld_pad=0),
               Case(f"gemv.mma.m{M}.swiglu", "gemv", M, 1536, 896, flags=EPI_SWIGLU, norm=True, ld_pad=0),
               Case(f"gemv.mma.m{M}.streamed", "gemv", M, 1024, 8192, flags=EPI_RESIDUAL, alias=True, ld_pad=0)]
    return cs


def gemv_reg_cases(sms: int) -> List[Case]:
    """shapes that put the register-streaming kernel at every wpi in {1, 2, 4, 8} and g in {1, 2, 4} (TL_GEMV_IMPL=reg)"""
    cs = []
    for K in (512, 2048, 4096, 8192):
        nvec = K // 8
        wpi = 1
        while wpi < 8 and -(-nvec // (32 * wpi)) > 4:
            wpi *= 2
        wave = sms * 2 * (8 // wpi)
        for g in (1, 2, 4):
            N = 2 * (4 * wave * g) if g > 1 else 2 * max(8, wave // 2)
            if N * K * 2 > (768 << 20):
                continue
            cs.append(Case(f"gemv.reg.k{K}.g{g}", "gemv", 3 if g == 4 else 1, N, K, flags=EPI_BIAS, ld_pad=0))
    return cs


def model_calls(cfg, prefill=300, gemv_rows=(1, 3), batched=(5, 64), train_tokens=2100, head_chunk=2048) -> List[Case]:
    """Every Linear call of the model for one config, with the shapes, flags, operand majors, workspace and aliasing of
    its call site."""
    H, I, Q, QKV, V = cfg.hidden, cfg.intermediate, cfg.q_dim, cfg.qkv_dim, cfg.vocab
    qb = EPI_BIAS if cfg.qkv_bias else 0
    cs = []

    def gemm(name, M, N, K, flags=0, **kw):
        cs.append(Case(f"{cfg.name}.{name}", "gemm", M, N, K, flags=flags, ld_pad=0, **kw))

    def gemv(name, M, N, K, flags=0, **kw):
        cs.append(Case(f"{cfg.name}.{name}", "gemv", M, N, K, flags=flags, ld_pad=0, **kw))

    T = prefill                                    # shard.py:275-283 (prefill, o / down in place on x)
    gemm(f"prefill{T}.qkv", T, QKV, H, qb)
    gemm(f"prefill{T}.o", T, H, Q, EPI_RESIDUAL, alias=True)
    gemm(f"prefill{T}.gu", T, 2 * I, H, EPI_SWIGLU)
    gemm(f"prefill{T}.down", T, H, I, EPI_RESIDUAL, alias=True)
    for B in batched:                              # shard.py:327-335 (batched decode: workspace, fused norm)
        ws = splitk_ws(min(B, 128), max(QKV, H))
        gemm(f"dec{B}.qkv", B, QKV, H, qb, ws_bytes=ws)
        gemm(f"dec{B}.o", B, H, Q, EPI_RESIDUAL, alias=True, ws_bytes=ws, norm=True)
        gemm(f"dec{B}.gu", B, 2 * I, H, EPI_SWIGLU, ws_bytes=ws)
        gemm(f"dec{B}.down", B, H, I, EPI_RESIDUAL, alias=True, ws_bytes=ws, norm=True)
        gemm(f"dec{B}.down_last", B, H, I, EPI_RESIDUAL, alias=True, ws_bytes=ws)
        gemm(f"dec{B}.head", B, V, H)              # stage.py:99 (logits_dec[:B])
    for m in gemv_rows:                            # shard.py:311-317 (GEMV decode with next_w), stage.py:68
        gemv(f"gemv{m}.qkv", m, QKV, H, qb, norm=True, next_w=True)
        gemv(f"gemv{m}.o", m, H, Q, EPI_RESIDUAL, alias=True, next_w=True)
        gemv(f"gemv{m}.gu", m, 2 * I, H, EPI_SWIGLU, norm=True, next_w=True)
        gemv(f"gemv{m}.down", m, H, I, EPI_RESIDUAL, alias=True, next_w=True)
        gemv(f"gemv{m}.head", m, V, H, norm=True)
    n = train_tokens                               # train.py:179-197 (forward), 311-337 (dgrad, wgrad)
    gemm(f"train{n}.qkv", n, QKV, H, qb)
    gemm(f"train{n}.o", n, H, Q, EPI_RESIDUAL)
    gemm(f"train{n}.gu", n, 2 * I, H)
    gemm(f"train{n}.down", n, H, I, EPI_RESIDUAL)
    gemm(f"train{n}.dgrad_down", n, I, H, B_MN)
    gemm(f"train{n}.dgrad_gu", n, H, 2 * I, B_MN)
    gemm(f"train{n}.dgrad_o", n, Q, H, B_MN)
    gemm(f"train{n}.dgrad_qkv", n, H, QKV, B_MN)
    for acc in (0, EPI_ACCUM):
        tag = "acc" if acc else "set"
        gemm(f"train{n}.wgrad_down.{tag}", H, I, n, A_MN | B_MN | acc)
        gemm(f"train{n}.wgrad_gu.{tag}", 2 * I, H, n, A_MN | B_MN | acc)
        gemm(f"train{n}.wgrad_o.{tag}", H, Q, n, A_MN | B_MN | acc)
        gemm(f"train{n}.wgrad_qkv.{tag}", QKV, H, n, A_MN | B_MN | acc)
    for a in range(0, n, head_chunk):              # train.py:233-245 (fused head, 2048-token chunks, ragged tail)
        k = min(n, a + head_chunk) - a
        gemm(f"head{n}@{a}.logits", k, V, H)
        gemm(f"head{n}@{a}.dgrad", k, H, V, B_MN)
        gemm(f"head{n}@{a}.wgrad", V, H, k, A_MN | B_MN | (EPI_ACCUM if a else 0))
    mb = 512                                       # train.py:224, 259, 358 (pipelined head: row slices of the stash)
    gemm(f"headpipe{mb}.logits", mb, V, H)
    gemm(f"headpipe{mb}.dgrad", mb, H, V, B_MN)
    gemm(f"headpipe{n}.wgrad", V, H, n, A_MN | B_MN)
    return cs
