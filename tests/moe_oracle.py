"""CPU oracle for Qwen3-MoE, restated from HF ``models/qwen3_moe/modeling_qwen3_moe.py`` (transformers 5.5) on top of the
dense oracle's attention and norms (oracle/shard_oracle.py).  TEST INFRASTRUCTURE ONLY.

The MoE block, per token, h = post_attention_layernorm(x):
  logits = bf16(h @ gate^T); p = softmax(fp32(logits)); top-k of p (renormalised when norm_topk_prob);
  for each picked expert in ascending index: a = bf16(silu(gate) * up), y = bf16(a @ down^T), c = bf16(fp32(y) * w),
  acc = bf16(acc + c) from +0;  out = bf16(x + acc).
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn.functional as F

from oracle import shard_oracle as O


def route(cfg, logits: torch.Tensor):
    """HF Qwen3MoeTopKRouter: ids [N,k] (torch.topk order) and fp32 weights."""
    p = F.softmax(logits, dtype=torch.float32, dim=-1)
    top, ids = torch.topk(p, cfg.top_k, dim=-1)
    if cfg.norm_topk_prob:
        top = top / top.sum(dim=-1, keepdim=True)
    return ids, top


def moe_block(cfg, sd: Dict[str, torch.Tensor], li: int, h: torch.Tensor) -> torch.Tensor:
    """HF Qwen3MoeSparseMoeBlock with eager experts: h [..., H] -> acc [..., H] (before the residual)."""
    p = f"model.layers.{li}.mlp."
    shape = h.shape
    h = h.reshape(-1, shape[-1])
    ids, w = route(cfg, F.linear(h, sd[p + "gate.weight"]))
    gu, dn = sd[p + "experts.gate_up_proj"], sd[p + "experts.down_proj"]
    acc = torch.zeros_like(h)
    for e in sorted(set(ids.flatten().tolist())):
        slot, tok = torch.where((ids == e).T)
        g, u = F.linear(h[tok], gu[e]).chunk(2, dim=-1)
        y = F.linear(F.silu(g) * u, dn[e])
        acc.index_add_(0, tok, (y * w[tok, slot, None]).to(acc.dtype))
    return acc.reshape(shape)


def decoder_layer(cfg, sd, w: O.LayerWeights, li: int, x, cos, sin, attn_mode="sdpa_math", cache=None):
    """oracle/shard_oracle.py ``decoder_layer`` with the MoE block in place of the dense MLP."""
    B, S, _ = x.shape
    d = cfg.head_dim
    h = O.rmsnorm(x, w.ln1, cfg.rms_eps)
    q = F.linear(h, w.wq, w.bq).view(B, S, -1, d)
    k = F.linear(h, w.wk, w.bk).view(B, S, -1, d)
    v = F.linear(h, w.wv, w.bv).view(B, S, -1, d)
    if cfg.qk_norm:
        q = O.rmsnorm(q, w.qn, cfg.rms_eps)
        k = O.rmsnorm(k, w.kn, cfg.rms_eps)
    q, k, v = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)
    q, k = O.apply_rope(q, k, cos, sin)
    if cache is not None:
        k, v = cache.update(li, k, v)
    fn = O.attention_eager if attn_mode == "eager" else O.attention_sdpa_math
    x = x + F.linear(fn(q, k, v, d ** -0.5, cfg.n_heads // cfg.n_kv_heads), w.wo)
    return x + moe_block(cfg, sd, li, O.rmsnorm(x, w.ln2, cfg.rms_eps))


class MoeOracleModel(O.OracleModel):
    """``OracleModel`` of a Qwen3-MoE config (same embed / shards / final norm / lm_head composition)."""

    def hidden(self, input_ids, n_shards: int = 1, cache: Optional[O.KVCache] = None, past_len: int = 0,
               per_layer=None):
        cfg = self.cfg
        B, S = input_ids.shape
        x = F.embedding(input_ids, self.embed)
        pos = torch.arange(past_len, past_len + S)[None].expand(B, -1)
        cos, sin = O.rope_tables(cfg, pos, x.dtype)
        for r in O.split_layers(cfg.n_layers, n_shards):
            for i in r:
                x = decoder_layer(cfg, self.sd, self.layers[i], i, x, cos, sin, self.attn_mode, cache)
                if per_layer is not None:
                    per_layer.append(x)
            if n_shards > 1:
                x = O.wire_hop(x)
        return x


def hf_model(cfg, sd):
    """HF ``Qwen3MoeForCausalLM`` (eager attention, eager experts, bf16) holding ``sd`` (as tests/hf_util.py does)."""
    from transformers import Qwen3MoeConfig, Qwen3MoeForCausalLM
    hc = Qwen3MoeConfig(vocab_size=cfg.vocab, hidden_size=cfg.hidden, intermediate_size=cfg.intermediate,
                        moe_intermediate_size=cfg.moe_intermediate, num_hidden_layers=cfg.n_layers,
                        num_attention_heads=cfg.n_heads, num_key_value_heads=cfg.n_kv_heads, head_dim=cfg.head_dim,
                        num_experts=cfg.n_experts, num_experts_per_tok=cfg.top_k, norm_topk_prob=cfg.norm_topk_prob,
                        decoder_sparse_step=1, mlp_only_layers=[], max_position_embeddings=cfg.max_pos,
                        rope_parameters={"rope_type": "default", "rope_theta": cfg.rope_theta}, rms_norm_eps=cfg.rms_eps,
                        tie_word_embeddings=cfg.tied, use_sliding_window=False, attention_bias=False,
                        attn_implementation="eager", experts_implementation="eager")
    m = Qwen3MoeForCausalLM(hc)
    inv = m.model.rotary_emb.inv_freq.clone()      # from_pretrained keeps this buffer fp32
    m = m.to(torch.bfloat16)
    m.model.rotary_emb.inv_freq = inv
    m.model.rotary_emb.original_inv_freq = inv.clone()
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    assert all("rotary" in k or "inv_freq" in k for k in missing), missing
    return m.eval()
