"""Checkpoint in / out in the Hugging Face layout (SURVEY.md §8 f-2).

The reference reads, per worker, only the tensors of its layer range out of the hub snapshot's safetensors files and
remaps their keys to the local module (/root/reference/tensorlink/ml/worker.py:542-638, key remap :602-606), and
gathers parameters back through ``parameters(distributed=True)`` (ml/module.py:577-650).  Here a stage asks a
``LazyCheckpoint`` for exactly the HF tensor names it owns — nothing else is read from disk — and
``save_checkpoint`` writes one ``model-XXXXX-of-YYYYY.safetensors`` per stage plus the index and ``config.json``, so
the directory loads back here, in the reference, or in ``transformers``.  An FP8 model (ml/fp8.py) reads and writes HF's
fine-grained FP8 layout: ``...weight`` in float8_e4m3fn, ``...weight_scale_inv`` per 128x128 block and a
``quantization_config`` in ``config.json``.
"""
from __future__ import annotations

import json
import os
from typing import Dict, Iterator

import torch

from . import fp8 as F8
from .configs import ShardModelConfig, check_moe, moe_fields

INDEX = "model.safetensors.index.json"
SINGLE = "model.safetensors"


def quantization_from_dir(path: str):
    """The checkpoint's ``quantization_config`` parsed by ``ml/fp8.parse_quantization_config`` (None for a bf16
    checkpoint); variants this project does not run raise NotImplementedError."""
    with open(os.path.join(path, "config.json")) as f:
        return F8.parse_quantization_config(json.load(f).get("quantization_config"))


def config_from_dir(path: str) -> ShardModelConfig:
    """``config.json`` (HF Qwen2 / Qwen3 causal LM, bf16 or HF's fine-grained FP8) -> ShardModelConfig.  An FP8
    ``quantization_config`` the project does not run raises NotImplementedError (``quantization_from_dir``)."""
    with open(os.path.join(path, "config.json")) as f:
        c = json.load(f)
    quantization_from_dir(path)
    mt = c.get("model_type", "")
    moe = moe_fields(mt, c.get)
    if mt not in ("qwen2", "qwen3", "qwen3_moe"):
        raise ValueError(f"{path}: model_type {mt!r} is not supported (qwen2 / qwen3 / qwen3_moe)")
    if moe and c.get("quantization_config"):
        raise NotImplementedError(f"{path}: FP8 Qwen3-MoE checkpoints are not supported")
    qk_norm = mt in ("qwen3", "qwen3_moe")
    n_h = int(c["num_attention_heads"])
    hd = int(c.get("head_dim") or c["hidden_size"] // n_h)
    theta = (c.get("rope_parameters") or {}).get("rope_theta", c.get("rope_theta", 1e6))
    cfg = ShardModelConfig(c.get("_name_or_path") or os.path.basename(os.path.normpath(path)), int(c["hidden_size"]),
                           int(c["intermediate_size"]), int(c["num_hidden_layers"]), n_h, int(c["num_key_value_heads"]), hd,
                           int(c["vocab_size"]), tied=bool(c.get("tie_word_embeddings", False)), qkv_bias=not qk_norm,
                           qk_norm=qk_norm, rope_theta=float(theta), rms_eps=float(c.get("rms_norm_eps", 1e-6)),
                           max_pos=int(c.get("max_position_embeddings", 32768)), **moe)
    check_moe(cfg)
    return cfg


def config_to_json(cfg: ShardModelConfig) -> dict:
    return {"architectures": ["Qwen3ForCausalLM" if cfg.qk_norm else "Qwen2ForCausalLM"],
            "model_type": "qwen3" if cfg.qk_norm else "qwen2", "hidden_size": cfg.hidden,
            "intermediate_size": cfg.intermediate, "num_hidden_layers": cfg.n_layers, "num_attention_heads": cfg.n_heads,
            "num_key_value_heads": cfg.n_kv_heads, "head_dim": cfg.head_dim, "vocab_size": cfg.vocab,
            "tie_word_embeddings": bool(cfg.tied), "rope_theta": cfg.rope_theta, "rms_norm_eps": cfg.rms_eps,
            "max_position_embeddings": cfg.max_pos, "hidden_act": "silu", "torch_dtype": "bfloat16",
            "attention_bias": bool(cfg.qkv_bias), "_name_or_path": cfg.name,
            **({"architectures": ["Qwen3MoeForCausalLM"], "model_type": "qwen3_moe", "num_experts": cfg.n_experts,
                "num_experts_per_tok": cfg.top_k, "moe_intermediate_size": cfg.moe_intermediate,
                "norm_topk_prob": bool(cfg.norm_topk_prob), "decoder_sparse_step": 1, "mlp_only_layers": []}
               if cfg.is_moe else {})}


def _per_expert(cfg: ShardModelConfig, sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """HF's fused in-memory expert tensors -> the per-expert names Qwen3-MoE checkpoints store."""
    if not cfg.is_moe:
        return sd
    out: Dict[str, torch.Tensor] = {}
    Ie = cfg.moe_intermediate
    for k, t in sd.items():
        if k.endswith("mlp.experts.gate_up_proj"):
            pre = k[:-len("gate_up_proj")]
            for e in range(cfg.n_experts):
                out[f"{pre}{e}.gate_proj.weight"] = t[e, :Ie].contiguous()
                out[f"{pre}{e}.up_proj.weight"] = t[e, Ie:].contiguous()
        elif k.endswith("mlp.experts.down_proj"):
            pre = k[:-len("down_proj")]
            for e in range(cfg.n_experts):
                out[f"{pre}{e}.down_proj.weight"] = t[e].contiguous()
        else:
            out[k] = t
    return out


class LazyCheckpoint:
    """Read-only mapping ``HF tensor name -> tensor`` over a directory of safetensors files; a tensor is read from
    disk when it is asked for (``safe_open(...).get_tensor``), so a stage touches only its own layer range."""

    def __init__(self, path: str):
        self.path = path
        idx = os.path.join(path, INDEX)
        if os.path.exists(idx):
            with open(idx) as f:
                self.where: Dict[str, str] = dict(json.load(f)["weight_map"])
        else:
            from safetensors import safe_open
            files = [SINGLE] if os.path.exists(os.path.join(path, SINGLE)) else \
                sorted(f for f in os.listdir(path) if f.endswith(".safetensors"))
            if not files:
                raise FileNotFoundError(f"{path}: no safetensors files")
            self.where = {}
            for fn in files:
                with safe_open(os.path.join(path, fn), framework="pt") as f:
                    for k in f.keys():
                        self.where[k] = fn
        self.bytes_read = 0
        self._open: Dict[str, object] = {}

    def __contains__(self, name: str) -> bool:
        return name in self.where

    def keys(self) -> Iterator[str]:
        return iter(self.where)

    def __getitem__(self, name: str) -> torch.Tensor:
        from safetensors import safe_open
        fn = self.where[name]                       # KeyError names the missing tensor
        h = self._open.get(fn)
        if h is None:
            h = self._open[fn] = safe_open(os.path.join(self.path, fn), framework="pt")
        t = h.get_tensor(name)
        self.bytes_read += t.numel() * t.element_size()
        return t


def save_checkpoint(dm, path: str, link=None) -> None:
    """Every rank writes its stage's tensors; rank 0 adds ``config.json`` and the index over all ranks' files."""
    from safetensors.torch import save_file
    link = link or dm.link
    os.makedirs(path, exist_ok=True)
    sd = _per_expert(dm.cfg, {k: v.detach().to("cpu").contiguous() for k, v in dm.stage.params.hf_state_dict().items()})
    if dm.cfg.tied and "lm_head.weight" in sd and "model.embed_tokens.weight" in sd:
        sd.pop("lm_head.weight")                    # tied: stored once, like HF
    fn = f"model-{link.rank + 1:05d}-of-{link.world:05d}.safetensors"
    save_file(sd, os.path.join(path, fn), metadata={"format": "pt"})
    maps = link.all_gather_object({k: fn for k in sd})
    sizes = link.all_gather_object(sum(v.numel() * v.element_size() for v in sd.values()))
    if link.rank == 0:
        weight_map: Dict[str, str] = {}
        for m in maps:
            for k, f in m.items():
                weight_map.setdefault(k, f)         # a tied head on the last rank does not shadow the embedding
        with open(os.path.join(path, INDEX), "w") as f:
            json.dump({"metadata": {"total_size": int(sum(sizes))}, "weight_map": weight_map}, f, indent=1)
        with open(os.path.join(path, "config.json"), "w") as f:
            c = config_to_json(dm.cfg)
            if getattr(dm, "quantization", None):
                c["quantization_config"] = F8.config_dict()
            json.dump(c, f, indent=1)
    link.barrier()
