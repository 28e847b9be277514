"""TEST-ONLY: the CPU oracle (oracle/shard_oracle.py) with HF's 2-D ``attention_mask`` for padded training batches.

Semantics (HF ``forward`` without ``position_ids``, and the label rule of ``tensorlink_b200.ml.train.train_forward``):
  * RoPE positions stay 0..S-1 in every row, padded or not;
  * pad keys get an additive mask on top of ``causal_mask``: a real query attends to the real keys of its row at or
    before it;
  * a query row with no such key (a left-pad row) outputs zeros, as the CUDA kernels do;
  * the loss ignores every label predicted from a pad position.
With ``attention_mask=None`` every function here is the plain oracle's.
"""
from typing import Optional

import torch
import torch.nn.functional as F

from oracle import shard_oracle as O
from tests.oracle_stage import OracleStage, OracleTrainer


def mask_shift_labels(shift: torch.Tensor, attention_mask: Optional[torch.Tensor]) -> torch.Tensor:
    """The shifted label at t becomes -100 where ``attention_mask[b, t] == 0``."""
    if attention_mask is None:
        return shift
    return shift.masked_fill(attention_mask.to(shift.device) == 0, -100)


def key_padding_mask(key_mask: torch.Tensor, dtype) -> torch.Tensor:
    """Additive [B,1,1,T]: 0 on real keys, the dtype's min on pad keys (``key_mask`` bool [B,T])."""
    m = torch.zeros(key_mask.shape[0], 1, 1, key_mask.shape[1], dtype=dtype)
    return m.masked_fill_(~key_mask[:, None, None, :], torch.finfo(dtype).min)


def rows_with_keys(key_mask: torch.Tensor, S: int, T: int) -> torch.Tensor:
    """bool [B,1,S,1]: the query row sees at least one real key at or before it."""
    causal_ok = torch.arange(T)[None, :] <= torch.arange(T - S, T)[:, None]
    return (key_mask[:, None, :] & causal_ok[None]).any(-1)[:, None, :, None]


def attention_eager(q, k, v, scaling: float, n_rep: int, key_mask: Optional[torch.Tensor] = None):
    if key_mask is None:
        return O.attention_eager(q, k, v, scaling, n_rep)
    k, v = O.repeat_kv(k, n_rep), O.repeat_kv(v, n_rep)
    S, T = q.shape[2], k.shape[2]
    w = torch.matmul(q, k.transpose(2, 3)) * scaling
    w = w + O.causal_mask(S, T, q.dtype) + key_padding_mask(key_mask, q.dtype)
    w = F.softmax(w, dim=-1, dtype=torch.float32).to(q.dtype)
    w = torch.where(rows_with_keys(key_mask, S, T), w, torch.zeros((), dtype=w.dtype))
    o = torch.matmul(w, v)
    return o.transpose(1, 2).contiguous().reshape(q.shape[0], S, -1)


def attention_sdpa_math(q, k, v, scaling: float, n_rep: int, key_mask: Optional[torch.Tensor] = None):
    if key_mask is None:
        return O.attention_sdpa_math(q, k, v, scaling, n_rep)
    dt = q.dtype
    k, v = O.repeat_kv(k, n_rep).to(torch.float32), O.repeat_kv(v, n_rep)
    S, T = q.shape[2], k.shape[2]
    s = torch.matmul(q.to(torch.float32), k.transpose(2, 3)) * scaling
    s = s + O.causal_mask(S, T, torch.float32) + key_padding_mask(key_mask, torch.float32)
    p = F.softmax(s, dim=-1)
    p = torch.where(rows_with_keys(key_mask, S, T), p, torch.zeros((), dtype=p.dtype))
    o = torch.matmul(p.to(dt).to(torch.float32), v.to(torch.float32)).to(dt)
    return o.transpose(1, 2).contiguous().reshape(q.shape[0], S, -1)


def decoder_layer(cfg, w: O.LayerWeights, x, cos, sin, attn_mode: str = "sdpa_math",
                  key_mask: Optional[torch.Tensor] = None):
    """``O.decoder_layer`` (no cache) with a per-row key mask."""
    if key_mask is None:
        return O.decoder_layer(cfg, w, x, cos, sin, attn_mode)
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
    fn = attention_eager if attn_mode == "eager" else attention_sdpa_math
    a = fn(q, k, v, d ** -0.5, cfg.n_heads // cfg.n_kv_heads, key_mask)
    x = x + F.linear(a, w.wo)
    return x + O.swiglu_mlp(O.rmsnorm(x, w.ln2, cfg.rms_eps), w.wg, w.wu, w.wd)


def shard_forward(cfg, layers, hidden_states, cos, sin, attn_mode: str = "sdpa_math",
                  key_mask: Optional[torch.Tensor] = None):
    for w in layers:
        hidden_states = decoder_layer(cfg, w, hidden_states, cos, sin, attn_mode, key_mask)
    return hidden_states


class MaskedOracleModel(O.OracleModel):
    """``OracleModel.hidden / logits / loss`` with an optional ``attention_mask`` ([B,S], no KV cache)."""

    def hidden(self, input_ids, n_shards: int = 1, attention_mask: Optional[torch.Tensor] = None):
        if attention_mask is None:
            return super().hidden(input_ids, n_shards)
        cfg = self.cfg
        B, S = input_ids.shape
        x = F.embedding(input_ids, self.embed)
        cos, sin = O.rope_tables(cfg, torch.arange(S)[None].expand(B, -1), x.dtype)
        km = attention_mask != 0
        for r in O.split_layers(cfg.n_layers, n_shards):
            x = shard_forward(cfg, [self.layers[i] for i in r], x, cos, sin, self.attn_mode, km)
            if n_shards > 1 and not x.requires_grad:
                x = O.wire_hop(x)
        return x

    def logits(self, input_ids, n_shards: int = 1, attention_mask: Optional[torch.Tensor] = None):
        x = self.hidden(input_ids, n_shards, attention_mask)
        return F.linear(O.rmsnorm(x, self.norm, self.cfg.rms_eps), self.head)

    def loss(self, input_ids, labels, n_shards: int = 1, attention_mask: Optional[torch.Tensor] = None):
        logits = self.logits(input_ids, n_shards, attention_mask)
        lf = logits.to(torch.float32)
        shift = mask_shift_labels(F.pad(labels, (0, 1), value=-100)[:, 1:], attention_mask)
        loss = F.cross_entropy(lf.reshape(-1, lf.shape[-1]), shift.reshape(-1), ignore_index=-100)
        return loss, logits


# ------------------------------------------------------------------------------------------ pipeline-stage twin

class PaddedOracleTrainer(OracleTrainer):
    """``OracleTrainer`` that takes per-row key starts like ``StageTrainer`` (``supports_kv_start``): keys below
    ``kv_start[b]`` are masked in every layer; positions stay 0..S-1."""

    supports_kv_start = True

    def forward_layers(self, mb, x, kv_start=None):
        if kv_start is None:
            return super().forward_layers(mb, x)
        cfg, st = self.cfg, self.st
        b, S, _ = x.shape
        xin = x.detach().clone().requires_grad_(True)
        cos, sin = O.rope_tables(cfg, torch.arange(S)[None].expand(b, -1), x.dtype)
        key_mask = torch.arange(S)[None, :] >= kv_start.cpu().long()[:, None]
        y = shard_forward(cfg, [st.layers[i] for i in st.layer_ids], xin, cos, sin, "sdpa_math", key_mask)
        self.ctx[mb] = {"xin": xin, "y": y, "b": b, "S": S}
        return y.detach()


class PaddedOracleStage(OracleStage):
    def make_trainer(self):
        return PaddedOracleTrainer(self)
