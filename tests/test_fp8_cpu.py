"""HF fine-grained FP8 checkpoints without a GPU: quantize / dequantize against HF's own conversion ops bit for bit, the
``quantization_config`` checks, and the per-row scale layout of the parameter arena."""
import json
import os
from types import SimpleNamespace

import pytest
import torch

from tensorlink_b200.ml import configs as C
from tensorlink_b200.ml import fp8 as F8
from tensorlink_b200.ml.checkpoint import config_from_dir, config_to_json, quantization_from_dir
from tensorlink_b200.ml.shard import ShardParams
from tensorlink_b200.ml.weights import init_state_dict

HF_QC = {"quant_method": "fp8", "fmt": "e4m3", "activation_scheme": "dynamic", "weight_block_size": [128, 128]}


def _hf_ops():
    from transformers.integrations.finegrained_fp8 import Fp8Dequantize, Fp8Quantize
    quantizer = SimpleNamespace(quantization_config=SimpleNamespace(weight_block_size=(128, 128)))
    return Fp8Quantize(quantizer), Fp8Dequantize(quantizer)


def _weight(shape, seed):
    """A bf16 weight whose blocks cover the edge cases: an all-zero block, a block whose amax sits on both signs, and a
    block with a tiny tail under a large amax (its codes land on e4m3 subnormals and zero)."""
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(shape, generator=g) * 0.02).to(torch.bfloat16)
    w[:128, :128] = 0
    if shape[0] >= 256:
        w[128:256, :128] = torch.randn(128, 128, generator=g).to(torch.bfloat16)
        w[128, 0], w[129, 1] = 3.0, -3.0                  # +-amax: clamps exactly at +-448
    w[:128, 128:256] = (torch.randn(128, 128, generator=g) * 1e-4).to(torch.bfloat16)
    w[0, 128] = 1.0                                       # the rest of the block is ~1e-4 of amax: subnormal codes
    return w


@pytest.mark.parametrize("cfg", [C.TINY_QWEN2, C.TINY_QWEN3], ids=lambda c: c.name)
def test_quantize_dequantize_equal_hf(cfg):
    quant, dequant = _hf_ops()
    shapes = {"q_proj": (cfg.q_dim, cfg.hidden), "k_proj": (cfg.kv_dim, cfg.hidden), "o_proj": (cfg.hidden, cfg.q_dim),
              "gate_proj": (cfg.intermediate, cfg.hidden), "down_proj": (cfg.hidden, cfg.intermediate)}
    n_sub = 0
    for i, (name, shape) in enumerate(shapes.items()):
        w = _weight(shape, i)
        q, inv = F8.quantize(w)
        ref = quant.convert({f"{name}.weight": [w]})
        assert torch.equal(q.view(torch.uint8), ref[f"{name}.weight"].view(torch.uint8)), name
        assert torch.equal(inv, ref[f"{name}.weight_scale_inv"]), name
        assert float(inv[0, 0]) == 1.0                               # all-zero block: scale 1
        assert q.float().abs().max() == 448.0
        codes = q.view(torch.uint8) & 0x7F
        n_sub += int(((codes > 0) & (codes < 8)).sum())              # exponent field 0: subnormal
        deq = dequant.convert({"weight$": [q], "weight_scale_inv": [inv]}, full_layer_name=f"{name}.weight")
        hf32 = deq[f"{name}.weight"]
        assert torch.equal(F8.dequantize(q, inv, torch.float32), hf32), name
        assert torch.equal(F8.dequantize(q, inv), hf32.to(torch.bfloat16)), name
    assert n_sub > 0


def _write_config(tmp_path, qc):
    c = config_to_json(C.TINY_QWEN3)
    if qc is not None:
        c["quantization_config"] = qc
    with open(os.path.join(tmp_path, "config.json"), "w") as f:
        json.dump(c, f)
    return str(tmp_path)


def test_config_from_dir_accepts_hf_fp8(tmp_path):
    d = _write_config(tmp_path, dict(HF_QC, modules_to_not_convert=["lm_head"]))
    assert config_from_dir(d).hidden == C.TINY_QWEN3.hidden
    assert quantization_from_dir(d) == {"block": 128}
    assert quantization_from_dir(_write_config(tmp_path, None)) is None


@pytest.mark.parametrize("change", [{"weight_block_size": [64, 64]}, {"weight_block_size": None},
                                    {"activation_scheme": "static"}, {"fmt": "e5m2"}, {"quant_method": "awq"},
                                    {"modules_to_not_convert": ["model.layers.0.mlp.down_proj"]}],
                         ids=["block64", "per_tensor", "static", "e5m2", "awq", "bf16_linear"])
def test_config_from_dir_rejects_variants(tmp_path, change):
    d = _write_config(tmp_path, dict(HF_QC, **change))
    with pytest.raises(NotImplementedError):
        config_from_dir(d)


def test_quantization_config_object():
    obj = SimpleNamespace(quant_method=SimpleNamespace(value="fp8"), fmt="e4m3", activation_scheme="dynamic",
                          weight_block_size=(128, 128), modules_to_not_convert=None)
    assert F8.parse_quantization_config(obj) == {"block": 128}
    assert F8.parse_quantization_config(None) is None


@pytest.mark.parametrize("cfg", [C.TINY_QWEN2, C.TINY_QWEN3], ids=lambda c: c.name)
def test_row_scales_follow_fusion_and_map_back(cfg):
    """Per-row scales of fused q/k/v and interleaved gate/up are HF's grid expanded row by row, and hf_state_dict
    returns HF's names, codes and grids unchanged."""
    sd = init_state_dict(cfg, 5, torch.bfloat16, "cpu", layers=[1], with_embed=False, with_head=False)
    quant, _ = _hf_ops()
    hf = dict(sd)
    for k in [k for k in sd if k.endswith("proj.weight")]:
        hf.update(quant.convert({k: [sd[k]]}))
    p = ShardParams(cfg, [1], False, False, "cpu", fp8=True)
    p.load_hf_state_dict(hf)
    pre = "model.layers.1."
    grid = lambda n: hf[pre + n + ".weight_scale_inv"]
    want_qkv = torch.cat([grid("self_attn.q_proj"), grid("self_attn.k_proj"), grid("self_attn.v_proj")]).repeat_interleave(128, 0)
    assert torch.equal(p.s["l1.wqkv"], want_qkv)
    sgu = p.s["l1.wgu"]
    assert torch.equal(sgu[0::2], grid("mlp.gate_proj").repeat_interleave(128, 0))
    assert torch.equal(sgu[1::2], grid("mlp.up_proj").repeat_interleave(128, 0))
    assert torch.equal(p.v["l1.wgu"][1::2].view(torch.uint8), hf[pre + "mlp.up_proj.weight"].view(torch.uint8))
    out = p.hf_state_dict()
    assert set(out) == set(hf)
    for k, t in hf.items():
        assert out[k].dtype == t.dtype, k
        a, b = (out[k].view(torch.uint8), t.view(torch.uint8)) if t.dtype == torch.float8_e4m3fn else (out[k], t)
        assert torch.equal(a, b), k
    # a bf16 state dict is quantized on load by HF's rule
    p2 = ShardParams(cfg, [1], False, False, "cpu", fp8=True)
    p2.load_hf_state_dict(sd)
    assert torch.equal(p2.q8.view(torch.uint8), p.q8.view(torch.uint8)) and torch.equal(p2.scales, p.scales)


def test_training_and_optimizer_raise():
    from tensorlink_b200.ml import DistributedModel
    with pytest.raises(NotImplementedError, match="training"):
        DistributedModel(C.TINY_QWEN2, quantization_config=HF_QC)
    with pytest.raises(NotImplementedError):
        DistributedModel(C.TINY_QWEN2, training=False, quantization_config=dict(HF_QC, activation_scheme="static"))
    with pytest.raises(NotImplementedError, match="training"):
        ShardParams(C.TINY_QWEN2, [0], False, False, "cpu", with_grad=True, fp8=True)


def test_fp8_gemv_rows_fit_the_register_kernel(monkeypatch):
    """Wide down projections (32B / 72B models) lower the FP8 GEMV's row threshold to what one pass of the
    register-streaming fallback holds in shared memory."""
    from dataclasses import replace
    from tensorlink_b200.ml import shard
    monkeypatch.setattr(shard, "_FP8_GEMV_MAX_ROWS", 4)
    assert shard.fp8_gemv_rows(C.QWEN25_7B) == 4 and shard.fp8_gemv_rows(C.QWEN3_8B) == 4
    for I in (25600, 27648, 29568):
        assert shard.fp8_gemv_rows(replace(C.QWEN25_7B, intermediate=I)) == 3
        assert 3 * I * 2 + 3 * 256 <= 200 * 1024 < 4 * I * 2 + 4 * 256


def test_hf_module_with_fp8_weights():
    """An HF module whose Linears already hold e4m3 codes is read as FP8 through its config's quantization_config;
    without one it raises instead of casting the codes to bf16."""
    from tensorlink_b200.ml import DistributedModel
    from tests.hf_util import hf_model
    cfg = C.TINY_QWEN2
    m = hf_model(cfg, init_state_dict(cfg, 3, torch.bfloat16, "cpu"))
    lin = m.model.layers[0].mlp.down_proj
    lin.weight = torch.nn.Parameter(lin.weight.detach().to(torch.float8_e4m3fn), requires_grad=False)
    with pytest.raises(NotImplementedError, match="quantization_config"):
        DistributedModel(m, training=False)
    m.config.quantization_config = dict(HF_QC, weight_block_size=[64, 64])
    with pytest.raises(NotImplementedError, match="weight_block_size"):
        DistributedModel(m, training=False)
    m.config.quantization_config = HF_QC
    with pytest.raises(NotImplementedError, match="training"):
        DistributedModel(m)
