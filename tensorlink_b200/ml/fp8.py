"""Hugging Face's fine-grained FP8 checkpoints (``FineGrainedFP8Config``), run weight-only.

Format: every decoder-layer Linear weight is ``float8_e4m3fn`` with an fp32 ``weight_scale_inv`` per 128x128 block, and
``config.json`` carries ``quantization_config = {"quant_method": "fp8", "fmt": "e4m3", "activation_scheme": "dynamic",
"weight_block_size": [128, 128]}``.  Norms, biases, the embedding and the lm_head stay in the model dtype.

Numeric contract: an FP8 model here computes exactly the bf16 model HF builds from the checkpoint with
``FineGrainedFP8Config(dequantize=True)``: each weight is ``bf16(float32(w) * scale_inv[block])`` (HF's
``Fp8Dequantize`` followed by the cast to the model dtype), and everything after that is the bf16 pipeline.  This
deliberately differs from HF's GPU ``FP8Linear``, which also quantizes the activations per 1x128 group (W8A8); those
results depend on the kernel HF dispatches to.  ``activation_scheme="dynamic"`` is therefore accepted and run
weight-only.

In the parameter arena the scales are stored per ROW: ``[N, K/128]``, one per (arena row, 128-column group).  q/k/v
fusion and the gate/up interleave break HF's 128-row blocks, so the loader expands HF's grid row by row and
``hf_state_dict`` takes every 128th row of each projection back.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

FP8_MAX = 448.0                # largest finite float8_e4m3fn
BLOCK = 128
LINEARS = ("wqkv", "wo", "wgu", "wd")          # the arena names of a decoder layer's quantized Linears
_DECODER_LINEAR_PARTS = ("layers", "self_attn", "mlp", "q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj",
                         "down_proj")


def parse_quantization_config(qc) -> Optional[dict]:
    """HF's ``quantization_config`` (a dict, or a ``FineGrainedFP8Config``-like object) -> {"block": 128}, or None when
    ``qc`` is None.  What this project does not run raises NotImplementedError: another ``quant_method``, another
    ``fmt``, per-tensor scales or another block size, ``activation_scheme="static"``, and a ``modules_to_not_convert``
    that keeps a decoder-layer Linear in bf16."""
    if qc is None:
        return None
    get = (lambda k, d=None: qc.get(k, d)) if isinstance(qc, dict) else (lambda k, d=None: getattr(qc, k, d))
    method = get("quant_method")
    method = getattr(method, "value", method)           # HF's QuantizationMethod enum
    if method != "fp8":
        raise NotImplementedError(f"quantization_config quant_method={method!r}: only HF's fine-grained 'fp8' is supported")
    fmt = get("fmt", "e4m3")
    if fmt != "e4m3":
        raise NotImplementedError(f"quantization_config fmt={fmt!r}: only e4m3 is supported")
    block = get("weight_block_size")
    if block is None or [int(b) for b in block] != [BLOCK, BLOCK]:
        raise NotImplementedError(f"quantization_config weight_block_size={block!r}: only [128, 128] blocks are supported "
                                  "(per-tensor scales are not)")
    act = get("activation_scheme", "dynamic")
    if act != "dynamic":
        raise NotImplementedError(f"quantization_config activation_scheme={act!r}: only 'dynamic' (run weight-only) is "
                                  "supported")
    for m in get("modules_to_not_convert") or []:
        if any(p in str(m) for p in _DECODER_LINEAR_PARTS):
            raise NotImplementedError(f"quantization_config modules_to_not_convert={m!r}: a decoder-layer Linear left in "
                                      "bf16 is not supported")
    return {"block": BLOCK}


def config_dict() -> dict:
    """The ``quantization_config`` written to ``config.json`` by ``save_pretrained``."""
    return {"quant_method": "fp8", "fmt": "e4m3", "activation_scheme": "dynamic", "weight_block_size": [BLOCK, BLOCK],
            "modules_to_not_convert": ["lm_head"]}


def _check_shape(w: torch.Tensor):
    R, C = w.shape
    if R % BLOCK or C % BLOCK:
        raise NotImplementedError(f"FP8 weight of shape {tuple(w.shape)}: both dimensions must be multiples of {BLOCK}")
    return R, C


def quantize(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """HF's ``Fp8Quantize`` on one [R, C] weight: per 128x128 block ``scale = 448 / amax`` (1 for an all-zero block),
    ``q = float8_e4m3fn(clamp(w * scale, -448, 448))``.  Returns (q [R, C], scale_inv [R/128, C/128] fp32)."""
    R, C = _check_shape(w)
    blocks = w.to(torch.float32).reshape(R // BLOCK, BLOCK, C // BLOCK, BLOCK)
    amax = blocks.abs().amax(dim=(1, 3))
    scale = FP8_MAX / torch.where(amax > 0, amax, torch.ones_like(amax))
    scale = torch.where(amax > 0, scale, torch.ones_like(scale))
    q = torch.clamp(blocks * scale[:, None, :, None], min=-FP8_MAX, max=FP8_MAX).to(torch.float8_e4m3fn)
    return q.reshape(R, C), (1.0 / scale).to(torch.float32)


def dequantize(q: torch.Tensor, scale_inv: torch.Tensor, dtype=torch.bfloat16) -> torch.Tensor:
    """HF's ``Fp8Dequantize`` (fp32 ``q * scale_inv`` per block) followed by the cast to ``dtype``."""
    R, C = _check_shape(q)
    blocks = q.to(torch.float32).reshape(R // BLOCK, BLOCK, C // BLOCK, BLOCK)
    return (blocks * scale_inv.reshape(R // BLOCK, 1, C // BLOCK, 1)).reshape(R, C).to(dtype)


def rows_from_grid(scale_inv: torch.Tensor) -> torch.Tensor:
    """[R/128, C/128] block grid -> [R, C/128] per-row scales (the arena's layout)."""
    return scale_inv.to(torch.float32).repeat_interleave(BLOCK, dim=0)


def grid_from_rows(rows: torch.Tensor) -> torch.Tensor:
    """[R, C/128] per-row scales of one projection (rows in HF order) -> HF's [R/128, C/128] grid."""
    return rows[::BLOCK].clone()
