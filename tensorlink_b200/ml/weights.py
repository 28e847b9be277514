"""Seeded random-init weights, HF parameter names, shared by the oracle and the CUDA shards.

The reference loads real checkpoints shard-by-shard from safetensors
(/root/reference/tensorlink/ml/worker.py:542-638, key remap ``layers.{local_idx}.`` at :602-606).
There is no network here, so every tensor is drawn from its own generator seeded by
(base_seed, parameter name): any rank can materialise exactly its layer range, and the CPU
oracle sees bit-identical values.  Biases and norm gains are deliberately non-trivial
(HF's default init would give bias = 0, gain = 1 and hide layout bugs).
"""
from __future__ import annotations

import zlib
from typing import Dict, Iterable, Optional

import torch

from .configs import ShardModelConfig

INIT_STD = 0.02


def _seed_for(base_seed: int, name: str) -> int:
    return (base_seed * 1_000_003 + zlib.crc32(name.encode())) & 0x7FFF_FFFF_FFFF


def _draw(base_seed: int, name: str, shape, mean: float, std: float, dtype, device) -> torch.Tensor:
    dev = torch.device(device)
    g = torch.Generator(device=dev if dev.type == "cuda" else "cpu")
    g.manual_seed(_seed_for(base_seed, name))
    t = torch.empty(shape, dtype=torch.float32, device=dev if dev.type == "cuda" else "cpu")
    t.normal_(mean, std, generator=g)
    return t.to(dtype=dtype, device=dev)


def layer_param_shapes(cfg: ShardModelConfig) -> Dict[str, tuple]:
    H, I = cfg.hidden, cfg.intermediate
    s = {
        "input_layernorm.weight": (H,),
        "self_attn.q_proj.weight": (cfg.q_dim, H),
        "self_attn.k_proj.weight": (cfg.kv_dim, H),
        "self_attn.v_proj.weight": (cfg.kv_dim, H),
        "self_attn.o_proj.weight": (H, cfg.q_dim),
        "post_attention_layernorm.weight": (H,),
    }
    if cfg.is_moe:
        # HF's in-memory (fused) expert layout; the checkpoints on disk hold one tensor per expert (ml/shard.py)
        E, Ie = cfg.n_experts, cfg.moe_intermediate
        s.update({"mlp.gate.weight": (E, H), "mlp.experts.gate_up_proj": (E, 2 * Ie, H),
                  "mlp.experts.down_proj": (E, H, Ie)})
    else:
        s.update({"mlp.gate_proj.weight": (I, H), "mlp.up_proj.weight": (I, H), "mlp.down_proj.weight": (H, I)})
    if cfg.qkv_bias:
        s["self_attn.q_proj.bias"] = (cfg.q_dim,)
        s["self_attn.k_proj.bias"] = (cfg.kv_dim,)
        s["self_attn.v_proj.bias"] = (cfg.kv_dim,)
    if cfg.qk_norm:
        s["self_attn.q_norm.weight"] = (cfg.head_dim,)
        s["self_attn.k_norm.weight"] = (cfg.head_dim,)
    return s


def _is_gain(name: str) -> bool:
    return name.endswith("norm.weight") or name.endswith("layernorm.weight")


def init_tensor(cfg: ShardModelConfig, name: str, shape, seed: int, dtype, device) -> torch.Tensor:
    if _is_gain(name):
        return _draw(seed, name, shape, 1.0, 0.1, dtype, device)
    return _draw(seed, name, shape, 0.0, INIT_STD, dtype, device)


def init_state_dict(cfg: ShardModelConfig, seed: int = 1234, dtype=torch.bfloat16,
                    device="cpu", layers: Optional[Iterable[int]] = None,
                    with_embed: bool = True, with_head: bool = True) -> Dict[str, torch.Tensor]:
    """HF-named state dict (``model.layers.N.…``) for the given layer subset."""
    sd: Dict[str, torch.Tensor] = {}
    if with_embed:
        n = "model.embed_tokens.weight"
        sd[n] = init_tensor(cfg, n, (cfg.vocab, cfg.hidden), seed, dtype, device)
    layer_ids = range(cfg.n_layers) if layers is None else layers
    for li in layer_ids:
        for short, shape in layer_param_shapes(cfg).items():
            n = f"model.layers.{li}.{short}"
            sd[n] = init_tensor(cfg, n, shape, seed, dtype, device)
    if with_head:
        n = "model.norm.weight"
        sd[n] = init_tensor(cfg, n, (cfg.hidden,), seed, dtype, device)
        if cfg.tied:
            e = "model.embed_tokens.weight"
            sd["lm_head.weight"] = sd[e] if e in sd else init_tensor(
                cfg, e, (cfg.vocab, cfg.hidden), seed, dtype, device)
        else:
            n = "lm_head.weight"
            sd[n] = init_tensor(cfg, n, (cfg.vocab, cfg.hidden), seed, dtype, device)
    return sd


def synthetic_tokens(cfg: ShardModelConfig, batch: int, seq: int, seed: int = 4321) -> torch.Tensor:
    """``randint(0, V, (B, S))`` int64 from a private generator (BASELINE.md §2)."""
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, cfg.vocab, (batch, seq), dtype=torch.int64, generator=g)
