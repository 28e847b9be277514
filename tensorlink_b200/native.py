"""ctypes binding of ``libtensorlink_b200.so`` (the C ABI in ``include/tensorlink_b200.h``).

There is no CPU fallback and no eager-PyTorch twin: if the library is missing, or no sm_90 (H100) device is
visible, every compute entry point raises.  PyTorch is used only to own device memory and streams.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_float, c_int, c_int32, c_size_t, c_void_p
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libtensorlink_b200.so")

EPI_BIAS, EPI_RESIDUAL, EPI_SWIGLU, EPI_OUT_F32, EPI_ACCUM, A_MN_MAJOR, B_MN_MAJOR = 1, 2, 4, 8, 16, 32, 64


class NativeError(RuntimeError):
    pass


# the trailing arguments of the score-log (_log) entry points: raw log, score log, column counter, n_cols, B_total, row0,
# stream
_LOG_ARGS = [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]
_WARP_ARGS = [c_float, c_float, c_float, c_float]      # min_p, typical_p, epsilon, eta

_SIGS = {
    "tl_abi_version": (c_int, []),
    "tl_last_error": (c_char_p, []),
    "tl_device_info": (c_int, [POINTER(c_int), POINTER(c_int), POINTER(c_int)]),
    "tl_rmsnorm_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p]),
    "tl_embed_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "tl_gemm_bf16": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                             c_void_p, c_void_p, c_int, c_void_p]),
    "tl_gemm_splitk_ws": (c_size_t, [c_int, c_int]),
    "tl_gemm_bf16_ws": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                                c_void_p, c_void_p, c_int, c_void_p, c_size_t, c_void_p]),
    "tl_gemm_bf16_ws_norm": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                                     c_void_p, c_void_p, c_int, c_void_p, c_size_t, c_void_p, c_float, c_void_p, c_void_p]),
    "tl_gemv_bf16": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                             c_float, c_int, c_void_p]),
    "tl_gemv_bf16_pf": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                c_float, c_int, c_void_p, c_size_t, c_void_p]),
    "tl_gemv_bf16_ctr": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                 c_float, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "tl_gemv_fp8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                            c_float, c_int, c_void_p]),
    "tl_gemv_fp8_ctr": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                                c_void_p, c_float, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "tl_dequant_fp8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "tl_rope_table": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "tl_rope_kv_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                               c_void_p, c_float, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "tl_attn_prefill_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                    c_int, c_int, c_int, c_float, c_void_p]),
    "tl_attn_decode_ws": (c_size_t, [c_int, c_int, c_int, c_int]),
    "tl_attn_decode_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_int,
                                   c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "tl_attn_decode_fused": (c_int, [c_void_p] * 9 + [c_float, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "tl_attn_verify_ws": (c_size_t, [c_int, c_int, c_int, c_int]),
    "tl_attn_verify_fwd": (c_int, [c_void_p] * 6 + [c_size_t, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "tl_prompt_lookup_draft": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "tl_prompt_lookup_accept": (c_int, [c_void_p] * 6 + [c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                                         c_void_p, c_int, c_void_p]),
    "tl_assist_prep": (c_int, [c_void_p, c_void_p, c_int] + [c_void_p] * 5),
    "tl_rope_kv_fwd_rows": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_float, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "tl_attn_prefill_fwd_rows": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                         c_int, c_int, c_int, c_float, c_void_p, c_void_p]),
    "tl_attn_decode_fwd_rows": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_int,
                                        c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p]),
    "tl_attn_decode_fused_rows": (c_int, [c_void_p] * 9 + [c_float, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p,
                                                           c_void_p]),
    "tl_decode_chain_ws": (c_size_t, [c_int, c_int, c_int, c_int]),
    "tl_decode_chain_geometry": (c_int, [c_int, c_int, c_int, c_void_p]),
    "tl_decode_chain_trace": (c_int, [c_void_p, c_int]),
    "tl_decode_chain": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p, c_size_t, c_void_p]),
    "tl_peer_alloc": (c_int, [c_size_t, POINTER(c_void_p), c_void_p]),
    "tl_peer_open": (c_int, [c_void_p, POINTER(c_void_p)]),
    "tl_peer_close": (c_int, [c_void_p]),
    "tl_peer_free": (c_int, [c_void_p]),
    "tl_peer_wait": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, ctypes.c_uint64, c_void_p, c_void_p]),
    "tl_peer_signal": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "tl_peer_put": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p]),
    "tl_lmhead_ws": (c_size_t, [c_int, c_int]),
    "tl_lmhead_argmax": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_void_p, c_size_t,
                                 c_int, c_int, c_int, c_void_p, c_void_p]),
    "tl_argmax_bf16": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_int, c_int, c_void_p]),
    "tl_argmax_bf16_log": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_int, c_int] + _LOG_ARGS),
    "tl_sample_ws": (c_size_t, [c_int]),
    "tl_sample": (c_int, [c_void_p, c_void_p, c_int, c_int, c_float, c_int, c_float, ctypes.c_uint64, c_void_p, c_void_p, c_size_t,
                          c_void_p] + _WARP_ARGS),
    "tl_sample_log": (c_int, [c_void_p, c_void_p, c_int, c_int, c_float, c_int, c_float, ctypes.c_uint64, c_void_p, c_void_p,
                              c_size_t] + _LOG_ARGS + _WARP_ARGS),
    "tl_spec_accept_ws": (c_size_t, [c_int]),
    "tl_spec_accept": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_float, c_int, c_float,
                               ctypes.c_uint64, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p] + _WARP_ARGS),
    "tl_logits_proc_ws": (c_size_t, [c_int, c_int]),
    "tl_history_fill": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "tl_argmax_proc": (c_int, [c_void_p] * 6 + [c_int, c_void_p, c_size_t, c_int, c_int, c_int, c_void_p]),
    "tl_sample_proc": (c_int, [c_void_p] * 6 + [c_int, c_int, c_int, c_int, c_float, c_int, c_float, ctypes.c_uint64, c_void_p,
                                                c_void_p, c_size_t, c_void_p] + _WARP_ARGS),
    "tl_argmax_proc_log": (c_int, [c_void_p] * 6 + [c_int, c_void_p, c_size_t, c_int, c_int, c_int] + _LOG_ARGS),
    "tl_sample_proc_log": (c_int, [c_void_p] * 6 + [c_int, c_int, c_int, c_int, c_float, c_int, c_float, ctypes.c_uint64,
                                                    c_void_p, c_void_p, c_size_t] + _LOG_ARGS + _WARP_ARGS),
    "tl_advance_pos": (c_int, [c_void_p, c_void_p, c_int, c_void_p]),
    "tl_append_token": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "tl_swiglu_fwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "tl_swiglu_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "tl_rmsnorm_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                               c_void_p]),
    "tl_rope_kv_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                               c_int, c_int, c_void_p]),
    "tl_qk_norm_bwd": (c_int, [c_void_p] * 6 + [c_float, c_int, c_int, c_int, c_int, c_void_p]),
    "tl_attn_bwd_ws": (c_size_t, [c_int, c_int, c_int]),
    "tl_attn_bwd": (c_int, [c_void_p] * 10 + [c_size_t, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "tl_attn_bwd_rows": (c_int, [c_void_p] * 10 + [c_size_t, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p,
                                                   c_void_p]),
    "tl_ce_fwd_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int, c_int, c_void_p]),
    "tl_embed_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "tl_colsum": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "tl_f32_to_bf16_accum": (c_int, [c_void_p, c_void_p, c_size_t, c_int, c_void_p]),
    "tl_add_inplace": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    "tl_scale_add_bf16": (c_int, [c_void_p, c_void_p, c_float, c_int, c_size_t, c_void_p]),
    "tl_scale_add_f32": (c_int, [c_void_p, c_void_p, c_float, c_int, c_size_t, c_void_p]),
    "tl_moe_max_tiles": (c_int, [c_int, c_int, c_int]),
    "tl_moe_route": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                             c_void_p, c_int, c_void_p]),
    "tl_moe_gather": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "tl_moe_gemm": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "tl_moe_combine": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "tl_moe_gemv": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                            c_void_p]),
    "tl_adamw_step": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_float, c_float, c_float, c_float,
                              c_float, c_int, c_int, c_void_p]),
}



class DecodeJob(ctypes.Structure):
    """``tl_decode_job`` (include/tensorlink_b200.h)."""
    _fields_ = [("type", c_int32), ("N", c_int32), ("K", c_int32), ("flags", c_int32),
                ("n_h", c_int32), ("n_kv", c_int32), ("d", c_int32), ("T_max", c_int32),
                ("eps", c_float), ("scale", c_float),
                ("W", c_void_p), ("x", c_void_p), ("y", c_void_p), ("bias", c_void_p), ("residual", c_void_p),
                ("norm_w", c_void_p), ("pos_dev", c_void_p), ("cos_tab", c_void_p), ("sin_tab", c_void_p),
                ("q_norm_w", c_void_p), ("k_norm_w", c_void_p), ("k_cache", c_void_p), ("v_cache", c_void_p)]


JOB_GEMV, JOB_ATTN = 0, 1
ATTN_POS_PER_ROW = 1
CHAIN_MAX_JOBS, CHAIN_SYNC_BYTES = 16, 1024
GEMV_COUNTER_WORDS = 4

_lib: Optional[ctypes.CDLL] = None


def load() -> ctypes.CDLL:
    """Load the shared library and bind every declared symbol (no device needed for this)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(tensorlink_b200 has no CPU or eager fallback)")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in _SIGS.items():
        fn = getattr(lib, name)       # AttributeError here = header/library mismatch
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def exported_symbols():
    return sorted(_SIGS)


def last_error() -> str:
    return (load().tl_last_error() or b"").decode()


def _check(rc: int, what: str):
    if rc != 0:
        raise NativeError(f"{what} failed ({rc}): {last_error()}")


_device_ok = False


def require_device():
    """Raise unless an H100-class (sm_90) device is current."""
    global _device_ok
    if _device_ok:
        return
    if not torch.cuda.is_available():
        raise NativeError("no CUDA device: the tensorlink_b200 shard executor runs on sm_90a only")
    sm, ma, mi = c_int(), c_int(), c_int()
    _check(load().tl_device_info(sm, ma, mi), "tl_device_info")
    _device_ok = True


def _p(t: Optional[torch.Tensor]) -> Optional[int]:
    if t is None:
        return None
    assert t.is_cuda, "device tensor expected"
    return t.data_ptr()


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)


def _stream() -> int:
    """The current CUDA stream of the current device as a raw handle (every launch asks: the C accessor costs ~0.1 us,
    ``torch.cuda.current_stream().cuda_stream`` builds a Python Stream object each time)."""
    if _raw_stream is not None:
        return _raw_stream(torch.cuda.current_device())
    return torch.cuda.current_stream().cuda_stream


def _bf16(*ts):
    for t in ts:
        if t is not None:
            assert t.dtype == torch.bfloat16 and t.is_contiguous(), (t.dtype, t.is_contiguous())


# ------------------------------------------------------------------------------------------ thin typed wrappers
def rmsnorm_fwd(x: torch.Tensor, w: torch.Tensor, eps: float, out: Optional[torch.Tensor] = None,
                rstd: Optional[torch.Tensor] = None) -> torch.Tensor:
    require_device()
    _bf16(x, w, out)
    H = x.shape[-1]
    rows = x.numel() // H
    out = torch.empty_like(x) if out is None else out
    _check(load().tl_rmsnorm_fwd(_p(x), _p(w), _p(out), _p(rstd), rows, H, eps, _stream()), "tl_rmsnorm_fwd")
    return out


def embed_fwd(ids: torch.Tensor, table: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    require_device()
    assert ids.dtype == torch.int64 and ids.is_contiguous()
    _bf16(table, out)
    V, H = table.shape
    n = ids.numel()
    out = torch.empty(*ids.shape, H, dtype=torch.bfloat16, device=table.device) if out is None else out
    _check(load().tl_embed_fwd(_p(ids), _p(table), _p(out), n, H, V, _stream()), "tl_embed_fwd")
    return out


def gemm_splitk_ws(M: int, N: int) -> int:
    return int(load().tl_gemm_splitk_ws(M, N))


def gemm(a: torch.Tensor, b: torch.Tensor, out: Optional[torch.Tensor] = None, *, bias=None, residual=None,
         flags: int = 0, M: Optional[int] = None, N: Optional[int] = None, K: Optional[int] = None,
         ws: Optional[torch.Tensor] = None, norm_w: Optional[torch.Tensor] = None, eps: float = 1e-6,
         h_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """C[M,N] = A·B^T with the epilogue ``flags``.  A is [M,K] (or [K,M] with A_MN_MAJOR), B is [N,K] (or [K,N])."""
    require_device()
    _bf16(a, b, bias, residual)
    a_mn, b_mn = bool(flags & A_MN_MAJOR), bool(flags & B_MN_MAJOR)
    if M is None:
        M = a.shape[1] if a_mn else a.shape[0]
    if K is None:
        K = a.shape[0] if a_mn else a.shape[1]
    if N is None:
        N = b.shape[1] if b_mn else b.shape[0]
    c_cols = N // 2 if flags & EPI_SWIGLU else N
    if out is None:
        out = torch.empty(M, c_cols, dtype=torch.float32 if flags & EPI_OUT_F32 else torch.bfloat16, device=a.device)
    if bias is not None:
        flags |= EPI_BIAS
    if residual is not None:
        flags |= EPI_RESIDUAL
    if norm_w is not None:          # also h_out = RMSNorm(out) * norm_w (fused into the split-K reduce when that path runs)
        assert h_out is not None and h_out.dtype == torch.bfloat16 and h_out.is_contiguous() and h_out.shape == out.shape
        _check(load().tl_gemm_bf16_ws_norm(_p(a), _p(b), _p(out), M, N, K, a.stride(0), b.stride(0), out.stride(0), _p(bias),
                                           _p(residual), flags, _p(ws), 0 if ws is None else ws.numel() * ws.element_size(),
                                           _p(norm_w), eps, _p(h_out), _stream()), "tl_gemm_bf16_ws_norm")
        return out
    if ws is not None:
        _check(load().tl_gemm_bf16_ws(_p(a), _p(b), _p(out), M, N, K, a.stride(0), b.stride(0), out.stride(0), _p(bias),
                                      _p(residual), flags, _p(ws), ws.numel() * ws.element_size(), _stream()),
               "tl_gemm_bf16_ws")
        return out
    _check(load().tl_gemm_bf16(_p(a), _p(b), _p(out), M, N, K, a.stride(0), b.stride(0), out.stride(0), _p(bias),
                               _p(residual), flags, _stream()), "tl_gemm_bf16")
    return out


_PREFETCH_BYTES = None


def prefetch_bytes() -> int:
    """How much of the next launch's weights a GEMV asks L2 to fetch (TL_PREFETCH_MB, default 8; 0 disables).  The next
    launch takes its rows in address order, so these are the bytes it reads first.  8 MB measured best on an H100 SXM
    (700 W) for Qwen2.5-7B decode: 4.89 ms per token against 4.93 at 16 MB and 5.00 at 26 MB, which covers the whole
    o projection; a larger prefetch competes with the current launch's own stream."""
    global _PREFETCH_BYTES
    if _PREFETCH_BYTES is None:
        _PREFETCH_BYTES = int(float(os.environ.get("TL_PREFETCH_MB", "8")) * (1 << 20))
    return _PREFETCH_BYTES


def gemv_counters(*shape, device=None) -> torch.Tensor:
    """Zeroed counter blocks for GEMV call sites that own one (``[*shape, GEMV_COUNTER_WORDS]`` int32): a captured graph
    keeps their addresses, and the kernels leave them zero."""
    return torch.zeros(*shape, GEMV_COUNTER_WORDS, dtype=torch.int32, device=device)


def gemv(x: torch.Tensor, w: torch.Tensor, out: Optional[torch.Tensor] = None, *, bias=None, residual=None,
         norm_w=None, eps: float = 1e-6, flags: int = 0, next_w: Optional[torch.Tensor] = None,
         counter: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``counter``: this call site's block from ``gemv_counters`` (decode call sites inside captured graphs); None
    takes one from the library's per-device pool."""
    require_device()
    _bf16(x, w, bias, residual, norm_w, out)
    M, K = x.shape
    N = w.shape[0]
    if out is None:
        out = torch.empty(M, N // 2 if flags & EPI_SWIGLU else N, dtype=torch.bfloat16, device=x.device)
    if bias is not None:
        flags |= EPI_BIAS
    if residual is not None:
        flags |= EPI_RESIDUAL
    nb = min(next_w.numel() * next_w.element_size(), prefetch_bytes()) if next_w is not None else 0
    _check(load().tl_gemv_bf16_ctr(_p(x), _p(w), _p(out), M, N, K, _p(bias), _p(residual), _p(norm_w), eps, flags,
                                   _p(counter), _p(next_w) if nb else None, nb, _stream()), "tl_gemv_bf16_ctr")
    return out


FP8_BLOCK = 128          # TL_FP8_BLOCK: columns per FP8 weight scale


def _fp8(w: torch.Tensor, scales: torch.Tensor):
    N, K = w.shape
    assert w.dtype == torch.float8_e4m3fn and w.is_contiguous(), (w.dtype, w.is_contiguous())
    assert scales.dtype == torch.float32 and scales.is_contiguous() and tuple(scales.shape) == (N, K // FP8_BLOCK), \
        (scales.dtype, tuple(scales.shape), (N, K // FP8_BLOCK))
    return N, K


def gemv_fp8(x: torch.Tensor, w: torch.Tensor, scales: torch.Tensor, out: Optional[torch.Tensor] = None, *, bias=None,
             residual=None, norm_w=None, eps: float = 1e-6, flags: int = 0, next_w: Optional[torch.Tensor] = None,
             counter: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``gemv`` over FP8 weights ``w`` [N,K] (float8_e4m3fn) with ``scales`` [N, K/128] fp32: the weight used is
    bf16(float(w) * scale), and the result equals ``gemv`` over ``dequant_fp8(w, scales)`` bit for bit."""
    require_device()
    _bf16(x, bias, residual, norm_w, out)
    N, K = _fp8(w, scales)
    M = x.shape[0]
    assert x.shape[1] == K, (tuple(x.shape), K)
    if out is None:
        out = torch.empty(M, N // 2 if flags & EPI_SWIGLU else N, dtype=torch.bfloat16, device=x.device)
    if bias is not None:
        flags |= EPI_BIAS
    if residual is not None:
        flags |= EPI_RESIDUAL
    nb = min(next_w.numel() * next_w.element_size(), prefetch_bytes()) if next_w is not None else 0
    _check(load().tl_gemv_fp8_ctr(_p(x), _p(w), _p(scales), _p(out), M, N, K, _p(bias), _p(residual), _p(norm_w), eps,
                                  flags, _p(counter), _p(next_w) if nb else None, nb, _stream()), "tl_gemv_fp8_ctr")
    return out


def dequant_fp8(w: torch.Tensor, scales: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """bf16 [N,K] = bf16(float(w) * scales[n][k/128]): HF's Fp8Dequantize followed by the cast to bf16.  ``out`` may be a
    larger scratch buffer: its first N*K elements are written and returned as [N,K]."""
    require_device()
    N, K = _fp8(w, scales)
    if out is None:
        out = torch.empty(N, K, dtype=torch.bfloat16, device=w.device)
    else:
        assert out.dtype == torch.bfloat16 and out.is_contiguous() and out.numel() >= N * K
        out = out.reshape(-1)[:N * K].view(N, K)
    _check(load().tl_dequant_fp8(_p(w), _p(scales), _p(out), N, K, _stream()), "tl_dequant_fp8")
    return out


def rope_table(inv_freq: torch.Tensor, max_pos: int):
    require_device()
    assert inv_freq.dtype == torch.float32 and inv_freq.is_cuda
    half = inv_freq.numel()
    cos = torch.empty(max_pos, half, dtype=torch.bfloat16, device=inv_freq.device)
    sin = torch.empty_like(cos)
    _check(load().tl_rope_table(_p(inv_freq), _p(cos), _p(sin), max_pos, half, _stream()), "tl_rope_table")
    return cos, sin


def _kv_start(kv_start, B):
    """``kv_start``: int32[>= B] on the device, row b's leading pad slots (include/tensorlink_b200.h, left-padded batches)"""
    if kv_start.dtype != torch.int32 or not kv_start.is_cuda or kv_start.numel() < B or not kv_start.is_contiguous():
        raise NativeError(f"kv_start must be a contiguous int32 CUDA tensor of at least {B} rows")


def rope_kv_fwd(qkv, q_out, k_cache, v_cache, pos0_dev, cos_tab, sin_tab, q_norm_w, k_norm_w, eps, S, n_h, n_kv, d,
                kv_start=None):
    """``kv_start`` (int32[B] device, optional): left-padded rows, through ``tl_rope_kv_fwd_rows``."""
    require_device()
    _bf16(qkv, q_out, k_cache, v_cache, cos_tab, sin_tab, q_norm_w, k_norm_w)
    n_tokens = qkv.shape[0]
    T_max = k_cache.shape[2]
    if kv_start is None:
        _check(load().tl_rope_kv_fwd(_p(qkv), _p(q_out), _p(k_cache), _p(v_cache), _p(pos0_dev), _p(cos_tab), _p(sin_tab),
                                     _p(q_norm_w), _p(k_norm_w), eps, n_tokens, S, n_h, n_kv, d, T_max, _stream()),
               "tl_rope_kv_fwd")
        return
    _kv_start(kv_start, n_tokens // S)
    _check(load().tl_rope_kv_fwd_rows(_p(qkv), _p(q_out), _p(k_cache), _p(v_cache), _p(pos0_dev), _p(cos_tab), _p(sin_tab),
                                      _p(q_norm_w), _p(k_norm_w), eps, n_tokens, S, n_h, n_kv, d, T_max, _p(kv_start),
                                      _stream()), "tl_rope_kv_fwd_rows")


def attn_prefill_fwd(q, k_cache, v_cache, out, lse, B, S, past_len, n_h, n_kv, d, scale, kv_start=None):
    require_device()
    _bf16(q, k_cache, v_cache, out)
    T_max = k_cache.shape[2]
    if kv_start is None:
        _check(load().tl_attn_prefill_fwd(_p(q), _p(k_cache), _p(v_cache), _p(out), _p(lse), B, S, past_len, n_h, n_kv, d,
                                          T_max, scale, _stream()), "tl_attn_prefill_fwd")
        return
    _kv_start(kv_start, B)
    _check(load().tl_attn_prefill_fwd_rows(_p(q), _p(k_cache), _p(v_cache), _p(out), _p(lse), B, S, past_len, n_h, n_kv, d,
                                           T_max, scale, _p(kv_start), _stream()), "tl_attn_prefill_fwd_rows")


def attn_decode_ws(B, n_h, d, T_max) -> int:
    return int(load().tl_attn_decode_ws(B, n_h, d, T_max))


def attn_decode_fwd(q, k_cache, v_cache, out, kv_len_dev, ws, B, n_h, n_kv, d, scale, kv_start=None):
    require_device()
    _bf16(q, k_cache, v_cache, out)
    T_max = k_cache.shape[2]
    if kv_start is None:
        _check(load().tl_attn_decode_fwd(_p(q), _p(k_cache), _p(v_cache), _p(out), _p(kv_len_dev), _p(ws),
                                         ws.numel() * ws.element_size(), B, n_h, n_kv, d, T_max, scale, _stream()),
               "tl_attn_decode_fwd")
        return
    _kv_start(kv_start, B)
    _check(load().tl_attn_decode_fwd_rows(_p(q), _p(k_cache), _p(v_cache), _p(out), _p(kv_len_dev), _p(ws),
                                          ws.numel() * ws.element_size(), B, n_h, n_kv, d, T_max, scale, _p(kv_start),
                                          _stream()), "tl_attn_decode_fwd_rows")


VERIFY_MAX_ROWS = 16


def attn_verify_ws(q_len, n_h, d, T_max) -> int:
    return int(load().tl_attn_verify_ws(q_len, n_h, d, T_max))


def attn_verify_fwd(q, k_cache, v_cache, out, pos_dev, ws, q_len, n_h, n_kv, d, scale):
    """q [q_len, n_h*d] at cache slots pos..pos+q_len-1 of row 0 (already appended) -> out [q_len, n_h*d]; query i sees
    keys 0..pos+i."""
    require_device()
    _bf16(q, k_cache, v_cache, out)
    assert pos_dev.dtype == torch.int32
    _check(load().tl_attn_verify_fwd(_p(q), _p(k_cache), _p(v_cache), _p(out), _p(pos_dev), _p(ws),
                                     ws.numel() * ws.element_size(), q_len, n_h, n_kv, d, k_cache.shape[2], scale, _stream()),
           "tl_attn_verify_fwd")


def lmhead_ws(M, V) -> int:
    return int(load().tl_lmhead_ws(M, V))


def lmhead_argmax(x, w, norm_w, eps, ids_out, logits_out, ws, counter: Optional[torch.Tensor] = None):
    """``counter``: the lm_head GEMV's block from ``gemv_counters``, or None for one from the library's pool."""
    require_device()
    _bf16(x, w, norm_w, logits_out)
    M, H = x.shape
    V = w.shape[0]
    assert ids_out.dtype == torch.int64
    _check(load().tl_lmhead_argmax(_p(x), _p(w), _p(norm_w), eps, _p(ids_out), _p(logits_out), _p(ws),
                                   ws.numel() * ws.element_size(), M, V, H,
                                   _p(counter), _stream()),
           "tl_lmhead_argmax")


def _log_args(log, M: int, V: int) -> list:
    """The score log ``(raw, scores, col, row0)`` as the _log entry points take it: raw / scores fp32 [n_cols, B_total, V]
    on the device (either may be None), col int32[2] {column, exit word}, launch row m logged at row row0 + m."""
    raw, scores, col, row0 = log
    ref = raw if raw is not None else scores
    if ref is None:
        raise NativeError("score log: neither a raw nor a score buffer")
    for t in (raw, scores):
        if t is not None and (t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous() or t.dim() != 3
                              or t.shape != ref.shape or t.shape[2] != V):
            raise NativeError(f"score log buffers must be contiguous fp32 CUDA tensors [n_cols, B_total, {V}] of one shape")
    if col is None:
        raise NativeError("score log: no column counter")
    _i32(col)
    if col.numel() < 2:
        raise NativeError("score log: the column counter is int32[2] {column, exit word}")
    return [_p(raw), _p(scores), _p(col), ref.shape[0], ref.shape[1], int(row0), _stream()]


def argmax_bf16(logits, ids_out, ws, log=None):
    """``log``: None, or a score log (``_log_args``) that receives the logits as raw values and as scores."""
    require_device()
    _bf16(logits)
    M, V = logits.shape
    if log is None:
        _check(load().tl_argmax_bf16(_p(logits), _p(ids_out), _p(ws), ws.numel() * ws.element_size(), M, V, _stream()),
               "tl_argmax_bf16")
        return
    _check(load().tl_argmax_bf16_log(_p(logits), _p(ids_out), _p(ws), ws.numel() * ws.element_size(), M, V,
                                     *_log_args(log, M, V)), "tl_argmax_bf16_log")


def sample_ws(M: int) -> int:
    return int(load().tl_sample_ws(M))


def _warp(min_p, typical_p, epsilon, eta):
    """The sampler's trailing warper arguments (include/tensorlink_b200.h; off at 0, 1, 0, 0)."""
    return float(min_p), float(typical_p), float(epsilon), float(eta)


def sample(logits, ids_out, counters, ws, temperature: float = 1.0, top_k: int = 0, top_p: float = 1.0, seed: int = 0,
           log=None, min_p: float = 0.0, typical_p: float = 1.0, epsilon: float = 0.0, eta: float = 0.0):
    """ids_out[m] ~ softmax(eta(epsilon(typical(min-p(top-p(top-k(logits[m] / temperature))))))); ``counters`` int32[M]
    advance by one per call.  ``log``: None, or a score log (``_log_args``): raw logits, and logits / temperature on the
    kept set, -inf elsewhere.  ``min_p`` / ``typical_p`` / ``epsilon`` / ``eta``: HF's MinP / Typical / Epsilon / Eta
    warpers, off at their defaults."""
    require_device()
    _bf16(logits)
    M, V = logits.shape
    assert ids_out.dtype == torch.int64 and counters.dtype == torch.int32 and counters.numel() >= M
    args = [_p(logits), _p(ids_out), M, V, float(temperature), int(top_k or 0), float(top_p), int(seed) & (2 ** 64 - 1),
            _p(counters), _p(ws), ws.numel() * ws.element_size()]
    warp = _warp(min_p, typical_p, epsilon, eta)
    if log is None:
        _check(load().tl_sample(*args, _stream(), *warp), "tl_sample")
    else:
        _check(load().tl_sample_log(*args, *_log_args(log, M, V), *warp), "tl_sample_log")


def spec_accept_ws(K: int) -> int:
    return int(load().tl_spec_accept_ws(K))


def spec_accept(p_logits, q_logits, in_ids, n_cand, counter, ids_out, ws, temperature: float = 1.0, top_k: int = 0,
                top_p: float = 1.0, seed: int = 0, min_p: float = 0.0, typical_p: float = 1.0, epsilon: float = 0.0,
                eta: float = 0.0):
    """Speculative sampling of one verify step: the target's rows p_logits [K+1, V_p], the assistant's q_logits [K, V_q]
    (both bf16, each warped as ``sample`` warps it), the drafts in_ids[1..n_cand] drawn from q -> ids_out[0..n] in
    ``pl_accept``'s form (the kept drafts, then the drawn token); ``counter`` int32[1] advances by one per call."""
    require_device()
    _bf16(p_logits, q_logits)
    K = q_logits.shape[0]
    if p_logits.shape[0] != K + 1:
        raise NativeError(f"spec_accept: {p_logits.shape[0]} target rows for {K} assistant rows (K+1 expected)")
    _i32(n_cand, counter)
    assert in_ids.dtype == torch.int64 and ids_out.dtype == torch.int64 and in_ids.numel() >= K + 1 and ids_out.numel() >= K + 1
    _check(load().tl_spec_accept(_p(p_logits), p_logits.shape[1], _p(q_logits), q_logits.shape[1], K, _p(in_ids), _p(n_cand),
                                 float(temperature), int(top_k or 0), float(top_p), int(seed) & (2 ** 64 - 1), _p(counter),
                                 _p(ids_out), _p(ws), ws.numel() * ws.element_size(), _stream(),
                                 *_warp(min_p, typical_p, epsilon, eta)), "tl_spec_accept")


LP_PENALTY, LP_NGRAM, LP_MIN_NEW, LP_PROMPT, LP_N_EOS, LP_EOS, LP_MAX_EOS = 0, 1, 2, 3, 4, 5, 8
LP_PARAMS = LP_EOS + LP_MAX_EOS
LP_BAN = 1


def logits_proc_ws(M: int, V: int) -> int:
    return int(load().tl_logits_proc_ws(M, V))


def _history(log, length, bits, M: int, V: int):
    """A token history (include/tensorlink_b200.h, logits processors): log int32 [>=M, L], len int32 [>=M], bits int32
    [>=M, ceil(V/32)] (the bitmap's words; torch has no uint32), all contiguous on the device."""
    for t in (log, length, bits):
        if t.dtype != torch.int32 or not t.is_cuda or not t.is_contiguous() or t.shape[0] < M:
            raise NativeError(f"history tensors must be contiguous int32 CUDA tensors of at least {M} rows")
    if bits.shape[1] != (V + 31) // 32:
        raise NativeError(f"history bitmap has {bits.shape[1]} words per row, V={V} needs {(V + 31) // 32}")
    return log.shape[1]


def history_fill(prompt, log, length, bits, V: int):
    """The history of row m becomes prompt[m] (int64 [M,S]): log[m, :S], len[m] = S and the presence bitmap."""
    require_device()
    assert prompt.dtype == torch.int64 and prompt.is_contiguous()
    M, S = prompt.shape
    L = _history(log, length, bits, M, V)
    _check(load().tl_history_fill(_p(prompt), _p(log), _p(length), _p(bits), M, S, L, V, _stream()), "tl_history_fill")


def argmax_proc(logits, ids_out, log, length, bits, params, ws, flags: int = 0, score_log=None):
    """ids_out[m] = torch.argmax of HF's processed fp32 scores of logits[m]; appends the id to row m's history.
    ``score_log``: None, or a score log (``_log_args``): raw logits and the processed scores."""
    require_device()
    _bf16(logits)
    M, V = logits.shape
    L = _history(log, length, bits, M, V)
    assert ids_out.dtype == torch.int64 and params.dtype == torch.int32 and params.numel() >= LP_PARAMS
    args = [_p(logits), _p(ids_out), _p(log), _p(length), _p(bits), _p(params), flags, _p(ws), ws.numel() * ws.element_size(),
            M, V, L]
    if score_log is None:
        _check(load().tl_argmax_proc(*args, _stream()), "tl_argmax_proc")
    else:
        _check(load().tl_argmax_proc_log(*args, *_log_args(score_log, M, V)), "tl_argmax_proc_log")


def sample_proc(logits, ids_out, log, length, bits, params, counters, ws, temperature: float = 1.0, top_k: int = 0,
                top_p: float = 1.0, seed: int = 0, flags: int = 0, score_log=None, min_p: float = 0.0, typical_p: float = 1.0,
                epsilon: float = 0.0, eta: float = 0.0):
    """``sample`` over HF's processed fp32 scores; appends the drawn id to row m's history.  ``score_log``: None, or a
    score log (``_log_args``): raw logits, and processed / temperature on the kept set, -inf elsewhere."""
    require_device()
    _bf16(logits)
    M, V = logits.shape
    L = _history(log, length, bits, M, V)
    assert ids_out.dtype == torch.int64 and counters.dtype == torch.int32 and counters.numel() >= M
    assert params.dtype == torch.int32 and params.numel() >= LP_PARAMS
    args = [_p(logits), _p(ids_out), _p(log), _p(length), _p(bits), _p(params), flags, M, V, L, float(temperature),
            int(top_k or 0), float(top_p), int(seed) & (2 ** 64 - 1), _p(counters), _p(ws), ws.numel() * ws.element_size()]
    warp = _warp(min_p, typical_p, epsilon, eta)
    if score_log is None:
        _check(load().tl_sample_proc(*args, _stream(), *warp), "tl_sample_proc")
    else:
        _check(load().tl_sample_proc_log(*args, *_log_args(score_log, M, V), *warp), "tl_sample_proc_log")


def lp_params(penalty: float, ngram: int, min_new: int, prompt_len: int, eos_ids) -> torch.Tensor:
    """The int32[LP_PARAMS] parameter block of the logits processors (host tensor; copy it to the device)."""
    import struct
    eos_ids = list(eos_ids)
    if len(eos_ids) > LP_MAX_EOS:
        raise NotImplementedError(f"min_new_tokens with more than {LP_MAX_EOS} EOS ids")
    p = [struct.unpack("<i", struct.pack("<f", float(penalty)))[0], int(ngram), int(min_new), int(prompt_len), len(eos_ids)]
    p += [int(e) for e in eos_ids] + [0] * (LP_MAX_EOS - len(eos_ids))
    return torch.tensor(p, dtype=torch.int32)


PL_NGRAM, PL_MAX_LEN, PL_N_EOS, PL_EOS, PL_MAX_EOS = 0, 1, 2, 3, 8
PL_PARAMS = PL_EOS + PL_MAX_EOS
PL_MAX_DRAFT = 15


def pl_params(ngram: int, max_length: int, eos_ids) -> torch.Tensor:
    """The int32[PL_PARAMS] parameter block of prompt-lookup decoding (host tensor; copy it to the device)."""
    eos_ids = list(eos_ids)
    if len(eos_ids) > PL_MAX_EOS:
        raise NotImplementedError(f"prompt lookup with more than {PL_MAX_EOS} EOS ids")
    p = [int(ngram), int(max_length), len(eos_ids)] + [int(e) for e in eos_ids] + [0] * (PL_MAX_EOS - len(eos_ids))
    return torch.tensor(p, dtype=torch.int32)


def _i32(*ts):
    for t in ts:
        if t.dtype != torch.int32 or not t.is_cuda or not t.is_contiguous():
            raise NativeError("contiguous int32 CUDA tensor expected")


def pl_draft(log, length, params, K: int, in_ids, n_cand):
    """Row 0's history (log int32 [L], length int32 [1]) -> in_ids int64 [K+1] (last token, drafts, filler), n_cand."""
    require_device()
    _i32(log, length, params, n_cand)
    assert in_ids.dtype == torch.int64 and in_ids.numel() >= K + 1 and params.numel() >= PL_PARAMS
    _check(load().tl_prompt_lookup_draft(_p(log), _p(length), log.shape[-1], _p(params), K, _p(in_ids), _p(n_cand),
                                         _stream()), "tl_prompt_lookup_draft")


def pl_accept(ids, in_ids, n_cand, log, length, bits, V: int, params, out_log, count, pos_dev, kv_len_dev, K: int):
    """The agreeing drafts of a verify step and the model's next token join the history and ``out_log``."""
    require_device()
    _i32(n_cand, log, length, params, count, pos_dev, kv_len_dev)
    assert ids.dtype == torch.int64 and in_ids.dtype == torch.int64 and out_log.dtype == torch.int64
    assert ids.numel() >= K + 1 and in_ids.numel() >= K + 1 and params.numel() >= PL_PARAMS
    if bits is not None and bits.shape[-1] != (V + 31) // 32:
        raise NativeError(f"history bitmap has {bits.shape[-1]} words per row, V={V} needs {(V + 31) // 32}")
    _check(load().tl_prompt_lookup_accept(_p(ids), _p(in_ids), _p(n_cand), _p(log), _p(length), _p(bits), log.shape[-1], V,
                                          _p(params), _p(out_log), _p(count), out_log.numel(), _p(pos_dev), _p(kv_len_dev),
                                          K, _stream()), "tl_prompt_lookup_accept")


def assist_prep(log, length, asst_in, in_ids, pos_dev, kv_len_dev):
    """Row 0's history (log int32 [L], length int32 [1], L >= 2 tokens) -> the assistant's 2-row catch-up input
    ``asst_in`` (the last two tokens) and positions (pos = kv_len = length - 2), and the target's in_ids[0]."""
    require_device()
    _i32(log, length, pos_dev, kv_len_dev)
    assert asst_in.dtype == torch.int64 and in_ids.dtype == torch.int64 and asst_in.numel() >= 2 and in_ids.numel() >= 1
    _check(load().tl_assist_prep(_p(log), _p(length), log.shape[-1], _p(asst_in), _p(in_ids), _p(pos_dev), _p(kv_len_dev),
                                 _stream()), "tl_assist_prep")


def advance_pos(pos_dev, kv_len_dev, delta: int):
    require_device()
    _check(load().tl_advance_pos(_p(pos_dev), _p(kv_len_dev), delta, _stream()), "tl_advance_pos")


def append_token(ids, out_tokens, step_dev):
    require_device()
    assert ids.dtype == torch.int64 and out_tokens.dtype == torch.int64 and out_tokens.is_contiguous()
    B, ld = out_tokens.shape
    _check(load().tl_append_token(_p(ids), _p(out_tokens), _p(step_dev), B, ld, _stream()), "tl_append_token")


# ------------------------------------------------------------------------------------------ peer-memory mailboxes
class _RawCuda:
    """A raw device allocation seen through ``__cuda_array_interface__`` (bytes), so torch can view it."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3,
                                         "strides": None}


def tensor_from_ptr(ptr: int, nbytes: int) -> torch.Tensor:
    """uint8 tensor over [ptr, ptr+nbytes) without taking ownership (the caller keeps the allocation alive).
    No target device is named: torch tags the view with the device that owns the memory (for a peer mapping, the
    neighbour's), and naming another one would silently turn the view into a copy.  Only ``data_ptr()`` of such a
    view is ever used (as a kernel argument); torch never launches work on it."""
    return torch.as_tensor(_RawCuda(ptr, nbytes))


def peer_alloc(nbytes: int):
    """(ptr, handle bytes[64]): zeroed device allocation exportable to other processes on this node."""
    require_device()
    ptr, h = c_void_p(), ctypes.create_string_buffer(64)
    _check(load().tl_peer_alloc(nbytes, ctypes.byref(ptr), h), "tl_peer_alloc")
    return ptr.value, bytes(h.raw)


def peer_open(handle: bytes) -> int:
    require_device()
    ptr = c_void_p()
    _check(load().tl_peer_open(ctypes.create_string_buffer(handle, 64), ctypes.byref(ptr)), "tl_peer_open")
    return ptr.value


def peer_close(ptr: int):
    _check(load().tl_peer_close(ptr), "tl_peer_close")


def peer_free(ptr: int):
    _check(load().tl_peer_free(ptr), "tl_peer_free")


def peer_wait(flag, want, err, wait_ns=None, timeout_ns: int = 0, bump=None):
    require_device()
    _check(load().tl_peer_wait(_p(flag), _p(want), _p(err), _p(wait_ns), timeout_ns, _p(bump), _stream()), "tl_peer_wait")


def peer_signal(flag_peer, sent, bump=None):
    require_device()
    _check(load().tl_peer_signal(_p(flag_peer), _p(sent), _p(bump), _stream()), "tl_peer_signal")


def peer_put(dst_peer, src, flag_peer, sent):
    require_device()
    nbytes = src.numel() * src.element_size()
    _check(load().tl_peer_put(_p(dst_peer), _p(src), nbytes, _p(flag_peer), _p(sent), _stream()), "tl_peer_put")


# ------------------------------------------------------------------------------------------ training wrappers
def swiglu_fwd(gu, h):
    require_device(); _bf16(gu, h)
    M, I = h.shape
    _check(load().tl_swiglu_fwd(_p(gu), _p(h), M, I, _stream()), "tl_swiglu_fwd")


def swiglu_bwd(gu, dh, dgu):
    require_device(); _bf16(gu, dh, dgu)
    M, I = dh.shape
    _check(load().tl_swiglu_bwd(_p(gu), _p(dh), _p(dgu), M, I, _stream()), "tl_swiglu_bwd")


def rmsnorm_bwd(x, w, dy, rstd, dx, dw_accum, dx_add=None):
    require_device(); _bf16(x, w, dy, dx, dx_add)
    H = x.shape[-1]
    _check(load().tl_rmsnorm_bwd(_p(x), _p(w), _p(dy), _p(rstd), _p(dx_add), _p(dx), _p(dw_accum), x.numel() // H, H,
                                 _stream()), "tl_rmsnorm_bwd")


def rope_kv_bwd(dq, dk, dv, dqkv, cos_tab, sin_tab, S, n_h, n_kv, d):
    require_device(); _bf16(dq, dk, dv, dqkv)
    _check(load().tl_rope_kv_bwd(_p(dq), _p(dk), _p(dv), _p(dqkv), _p(cos_tab), _p(sin_tab), dqkv.shape[0], S, n_h, n_kv,
                                 d, dk.shape[2], _stream()), "tl_rope_kv_bwd")


def attn_bwd_ws(B, S, n_h) -> int:
    return int(load().tl_attn_bwd_ws(B, S, n_h))


def attn_bwd(q, k_cache, v_cache, out, dout, lse, dq, dk, dv, ws, B, S, n_h, n_kv, d, scale, kv_start=None):
    """``kv_start`` (int32[B] device, optional): left-padded rows, through ``tl_attn_bwd_rows``."""
    require_device(); _bf16(q, k_cache, v_cache, out, dout, dq, dk, dv)
    if kv_start is None:
        _check(load().tl_attn_bwd(_p(q), _p(k_cache), _p(v_cache), _p(out), _p(dout), _p(lse), _p(dq), _p(dk), _p(dv), _p(ws),
                                  ws.numel() * ws.element_size(), B, S, n_h, n_kv, d, k_cache.shape[2], scale, _stream()),
               "tl_attn_bwd")
        return
    _kv_start(kv_start, B)
    _check(load().tl_attn_bwd_rows(_p(q), _p(k_cache), _p(v_cache), _p(out), _p(dout), _p(lse), _p(dq), _p(dk), _p(dv),
                                   _p(ws), ws.numel() * ws.element_size(), B, S, n_h, n_kv, d, k_cache.shape[2], scale,
                                   _p(kv_start), _stream()), "tl_attn_bwd_rows")


def ce_fwd_bwd(logits, labels, loss_sum, n_valid, dlogits, grad_scale: float):
    require_device(); _bf16(logits, dlogits)
    M, V = logits.shape
    assert labels.dtype == torch.int64 and loss_sum.dtype == torch.float32
    _check(load().tl_ce_fwd_bwd(_p(logits), _p(labels), _p(loss_sum), _p(n_valid), _p(dlogits), grad_scale, M, V,
                                _stream()), "tl_ce_fwd_bwd")


def embed_bwd(ids, dout, dtable):
    require_device(); _bf16(dout, dtable)
    V, H = dtable.shape
    _check(load().tl_embed_bwd(_p(ids), _p(dout), _p(dtable), ids.numel(), H, V, _stream()), "tl_embed_bwd")


def colsum(dy, db_accum):
    require_device()
    assert db_accum.dtype == torch.float32
    M, N = dy.shape
    _check(load().tl_colsum(_p(dy), _p(db_accum), M, N, dy.stride(0), _stream()), "tl_colsum")


def f32_to_bf16_accum(src, dst, accumulate: bool):
    require_device()
    _check(load().tl_f32_to_bf16_accum(_p(src), _p(dst), src.numel(), int(accumulate), _stream()), "tl_f32_to_bf16_accum")


def add_inplace(a, b):
    require_device(); _bf16(a, b)
    _check(load().tl_add_inplace(_p(a), _p(b), a.numel(), _stream()), "tl_add_inplace")


def scale_add(a, b, scale: float, accumulate: bool = True):
    """a = (a if accumulate else 0) + scale * b   (bf16 or fp32 pairs, same shape)."""
    require_device()
    assert a.dtype == b.dtype and a.numel() == b.numel() and a.is_contiguous() and b.is_contiguous()
    if a.dtype == torch.bfloat16:
        _check(load().tl_scale_add_bf16(_p(a), _p(b), scale, int(accumulate), a.numel(), _stream()), "tl_scale_add_bf16")
    else:
        assert a.dtype == torch.float32
        _check(load().tl_scale_add_f32(_p(a), _p(b), scale, int(accumulate), a.numel(), _stream()), "tl_scale_add_f32")


def adamw_step(param, grad, m, v, lr, beta1, beta2, eps, wd, step: int, decoupled: bool):
    require_device()
    _check(load().tl_adamw_step(_p(param), _p(grad), _p(m), _p(v), param.numel(), lr, beta1, beta2, eps, wd, step,
                                int(decoupled), _stream()), "tl_adamw_step")


def attn_decode_fused(qkv, k_cache, v_cache, out, pos_dev, cos_tab, sin_tab, q_norm_w, k_norm_w, eps, B, n_h, n_kv, d, scale,
                      kv_start=None):
    require_device(); _bf16(qkv, k_cache, v_cache, out)
    if kv_start is None:
        _check(load().tl_attn_decode_fused(_p(qkv), _p(k_cache), _p(v_cache), _p(out), _p(pos_dev), _p(cos_tab), _p(sin_tab),
                                           _p(q_norm_w), _p(k_norm_w), eps, B, n_h, n_kv, d, k_cache.shape[2], scale, _stream()),
               "tl_attn_decode_fused")
        return
    _kv_start(kv_start, B)
    _check(load().tl_attn_decode_fused_rows(_p(qkv), _p(k_cache), _p(v_cache), _p(out), _p(pos_dev), _p(cos_tab), _p(sin_tab),
                                            _p(q_norm_w), _p(k_norm_w), eps, B, n_h, n_kv, d, k_cache.shape[2], scale,
                                            _p(kv_start), _stream()), "tl_attn_decode_fused_rows")


def decode_chain_ws(M: int, n_h: int, n_kv: int, d: int) -> int:
    return int(load().tl_decode_chain_ws(M, n_h, n_kv, d))


def decode_chain_geometry(M: int, k_max: int, stage_kb: int = -1) -> Optional[tuple]:
    """(slot bytes, slots, consumer warps, K chunk) of the ring tl_decode_chain builds for M rows and a widest GEMV
    K of k_max, or None when it cannot place that shape.  stage_kb < 0: the process's TL_CHAIN_STAGE_KB.  Host only."""
    out = (ctypes.c_int * 4)()
    if load().tl_decode_chain_geometry(M, k_max, stage_kb, ctypes.cast(out, c_void_p)) != 0:
        return None
    return tuple(out)


CHAIN_TRACE_WORDS = 2 * (CHAIN_MAX_JOBS + 1) * 4 + CHAIN_MAX_JOBS * 160 + CHAIN_MAX_JOBS * 4


def decode_chain_trace(buf: Optional[torch.Tensor]):
    """``buf``: int64 [n_slots, CHAIN_TRACE_WORDS] (or None to switch tracing off)."""
    _check(load().tl_decode_chain_trace(_p(buf), 0 if buf is None else buf.shape[0]), "tl_decode_chain_trace")


def make_job(type_, **kw) -> DecodeJob:
    j = DecodeJob()
    j.type = type_
    for k, v in kw.items():
        if isinstance(v, torch.Tensor):
            v = v.data_ptr()
        setattr(j, k, v)
    return j


class DecodeChain:
    """One launch site of ``tl_decode_chain``: a host job array (kept alive here: a captured graph holds the parameter
    copy, eager launches re-read this array), the rows per step, the private sync slot and the prefetch hint."""

    def __init__(self, jobs, M: int, sync_slot: torch.Tensor, attn_ws: torch.Tensor, next_w: Optional[torch.Tensor] = None):
        assert 1 <= len(jobs) <= CHAIN_MAX_JOBS
        self.n, self.M = len(jobs), M
        self.host = (DecodeJob * self.n)(*jobs)
        self.sync_slot, self.attn_ws, self.next_w = sync_slot, attn_ws, next_w
        assert sync_slot.numel() * sync_slot.element_size() >= CHAIN_SYNC_BYTES

    def launch(self):
        require_device()
        nb = 0
        if self.next_w is not None and prefetch_bytes() > 0:
            nb = min(self.next_w.numel() * self.next_w.element_size(), prefetch_bytes())
        _check(load().tl_decode_chain(ctypes.cast(self.host, c_void_p), self.n, self.M, _p(self.sync_slot), _p(self.attn_ws),
                                      self.attn_ws.numel() * self.attn_ws.element_size(), _p(self.next_w) if nb else None, nb,
                                      _stream()), "tl_decode_chain")


def qk_norm_bwd(qkv_pre, dqkv, qn, kn, dqn_acc, dkn_acc, eps, n_h, n_kv, d):
    require_device(); _bf16(qkv_pre, dqkv, qn, kn)
    _check(load().tl_qk_norm_bwd(_p(qkv_pre), _p(dqkv), _p(qn), _p(kn), _p(dqn_acc), _p(dkn_acc), eps, dqkv.shape[0], n_h,
                                 n_kv, d, _stream()), "tl_qk_norm_bwd")


# ---------------------------------------------------------------------------------------------- Qwen3-MoE (csrc/moe.cu)
def moe_max_tiles(N: int, E: int, k: int) -> int:
    """128-row M-tiles the grouped GEMM of N tokens may need (every non-empty expert segment padded to a tile)."""
    return int(load().tl_moe_max_tiles(N, E, k))


def moe_route(logits: torch.Tensor, k: int, norm_topk: bool, ids: torch.Tensor, wts: torch.Tensor, plan=None):
    """Top-k routing of ``logits`` [N,E] bf16 into ``ids`` [N,k] int32 (ascending) and ``wts`` [N,k] fp32.  ``plan``:
    (counts [E], offsets [E+1], row_of [N*k], tiles [T,2]) int32 tensors for the grouped GEMM, or None."""
    require_device()
    _bf16(logits)
    N, E = logits.shape
    assert ids.dtype == torch.int32 and wts.dtype == torch.float32
    counts, offsets, row_of, tiles = plan if plan is not None else (None, None, None, None)
    _check(load().tl_moe_route(_p(logits), N, E, k, int(bool(norm_topk)), _p(ids), _p(wts), _p(counts), _p(offsets),
                               _p(row_of), _p(tiles), 0 if tiles is None else tiles.shape[0], _stream()), "tl_moe_route")


def moe_gather(h: torch.Tensor, row_of: torch.Tensor, hg: torch.Tensor, k: int):
    require_device()
    _bf16(h, hg)
    _check(load().tl_moe_gather(_p(h), _p(row_of), _p(hg), h.shape[0], k, h.shape[1], _stream()), "tl_moe_gather")
    return hg


def moe_gemm(a: torch.Tensor, w: torch.Tensor, out: torch.Tensor, tiles: torch.Tensor, flags: int = 0):
    """Grouped GEMM: ``w`` [E, N, K]; M-tile t of ``a`` [tiles*128, K] runs on expert tiles[t, 0]."""
    require_device()
    _bf16(a, w, out)
    E, N, K = w.shape
    _check(load().tl_moe_gemm(_p(a), _p(w), _p(out), _p(tiles), tiles.shape[0], E, N, K, out.stride(0), flags, _stream()),
           "tl_moe_gemm")
    return out


def moe_combine(y: torch.Tensor, row_of: torch.Tensor, wts: torch.Tensor, x: torch.Tensor, out: torch.Tensor):
    require_device()
    _bf16(y, x, out)
    N, k = wts.shape
    _check(load().tl_moe_combine(_p(y), _p(row_of), _p(wts), _p(x), _p(out), N, k, x.shape[1], _stream()), "tl_moe_combine")
    return out


def moe_gemv(x: torch.Tensor, w: torch.Tensor, out: torch.Tensor, ids: torch.Tensor, *, wts=None, residual=None,
             flags: int = EPI_SWIGLU):
    """Expert GEMV over the picked experts ``ids`` [M,k] of ``w`` [E, N, K] (see tl_moe_gemv)."""
    require_device()
    _bf16(x, w, out, residual)
    E, N, K = w.shape
    M, k = ids.shape
    _check(load().tl_moe_gemv(_p(x), _p(w), _p(out), _p(ids), _p(wts), _p(residual), M, k, N, K, flags, _stream()),
           "tl_moe_gemv")
    return out
