"""Hard-coded model constants for the shard executor (no config.json is reachable offline).

The reference resolves these through ``AutoConfig.from_pretrained`` on the HF hub
(/root/reference/tensorlink/ml/utils.py:890-916 ``load_model_skeleton``); here they are the
public model-card values from SURVEY.md §8 and the parameter counts are asserted in the tests.
"""
from __future__ import annotations

from dataclasses import dataclass, replace


@dataclass(frozen=True)
class ShardModelConfig:
    name: str
    hidden: int          # H
    intermediate: int    # I
    n_layers: int        # L
    n_heads: int         # n_h
    n_kv_heads: int      # n_kv
    head_dim: int        # d
    vocab: int           # V
    tied: bool           # lm_head shares embed_tokens
    qkv_bias: bool       # Qwen2: yes, Qwen3: no
    qk_norm: bool        # Qwen3: per-head RMSNorm on q/k before RoPE
    rope_theta: float = 1.0e6
    rms_eps: float = 1.0e-6
    max_pos: int = 32768
    # Qwen3-MoE (HF ``qwen3_moe``): every decoder layer's MLP is a router over ``n_experts`` SwiGLU experts of width
    # ``moe_intermediate``, ``top_k`` of them per token.  n_experts == 0: dense (``intermediate`` is the MLP width).
    n_experts: int = 0
    top_k: int = 0
    moe_intermediate: int = 0
    norm_topk_prob: bool = False

    @property
    def is_moe(self) -> bool:
        return self.n_experts > 0

    @property
    def q_dim(self) -> int:
        return self.n_heads * self.head_dim

    @property
    def kv_dim(self) -> int:
        return self.n_kv_heads * self.head_dim

    @property
    def qkv_dim(self) -> int:
        return self.q_dim + 2 * self.kv_dim

    def layer_matmul_params(self) -> int:
        """P_mm of SURVEY.md §8(d): matmul weights of one decoder layer (a MoE layer: the router and every expert)."""
        attn = self.hidden * self.qkv_dim + self.q_dim * self.hidden
        if self.is_moe:
            return attn + self.n_experts * self.hidden + self.n_experts * 3 * self.hidden * self.moe_intermediate
        return attn + 3 * self.hidden * self.intermediate

    def layer_params(self) -> int:
        p = self.layer_matmul_params() + 2 * self.hidden
        if self.qkv_bias:
            p += self.qkv_dim
        if self.qk_norm:
            p += 2 * self.head_dim
        return p

    def total_params(self) -> int:
        p = self.n_layers * self.layer_params() + self.vocab * self.hidden + self.hidden
        if not self.tied:
            p += self.vocab * self.hidden
        return p

    def active_params(self) -> int:
        """Parameters one token reads: ``total_params()`` with only ``top_k`` experts of each MoE layer (rooflines)."""
        if not self.is_moe:
            return self.total_params()
        idle = (self.n_experts - self.top_k) * 3 * self.hidden * self.moe_intermediate
        return self.total_params() - self.n_layers * idle

    def scaled(self, **kw) -> "ShardModelConfig":
        return replace(self, **kw)


QWEN25_05B = ShardModelConfig("Qwen/Qwen2.5-0.5B", 896, 4864, 24, 14, 2, 64, 151936,
                              tied=True, qkv_bias=True, qk_norm=False)
QWEN25_7B = ShardModelConfig("Qwen/Qwen2.5-7B", 3584, 18944, 28, 28, 4, 128, 152064,
                             tied=False, qkv_bias=True, qk_norm=False)
QWEN25_7B_INSTRUCT = replace(QWEN25_7B, name="Qwen/Qwen2.5-7B-Instruct")
QWEN3_8B = ShardModelConfig("Qwen/Qwen3-8B", 4096, 12288, 36, 32, 8, 128, 151936,
                            tied=False, qkv_bias=False, qk_norm=True, max_pos=40960)

# Small same-architecture configs used by parity tests (oracle finishes in seconds on CPU).
TINY_QWEN2 = ShardModelConfig("tiny-qwen2", 256, 768, 4, 4, 2, 64, 1024,
                              tied=True, qkv_bias=True, qk_norm=False, max_pos=4096)
TINY_QWEN2_D128 = ShardModelConfig("tiny-qwen2-d128", 512, 1536, 4, 4, 2, 128, 2048,
                                   tied=False, qkv_bias=True, qk_norm=False, max_pos=4096)
TINY_QWEN3 = ShardModelConfig("tiny-qwen3", 512, 1024, 4, 4, 2, 128, 2048,
                              tied=False, qkv_bias=False, qk_norm=True, max_pos=4096)

# Qwen3-MoE: ``intermediate`` keeps config.json's (unused) dense width so the config round-trips
QWEN3_30B_A3B = ShardModelConfig("Qwen/Qwen3-30B-A3B", 2048, 6144, 48, 32, 4, 128, 151936, tied=False, qkv_bias=False,
                                 qk_norm=True, max_pos=40960, n_experts=128, top_k=8, moe_intermediate=768,
                                 norm_topk_prob=True)
TINY_QWEN3_MOE = ShardModelConfig("tiny-qwen3-moe", 512, 1024, 4, 4, 2, 128, 2048, tied=False, qkv_bias=False,
                                  qk_norm=True, max_pos=4096, n_experts=32, top_k=4, moe_intermediate=256,
                                  norm_topk_prob=True)
TINY_QWEN3_MOE_UNNORM = replace(TINY_QWEN3_MOE, name="tiny-qwen3-moe-unnorm", norm_topk_prob=False)

REGISTRY = {c.name: c for c in (QWEN25_05B, QWEN25_7B, QWEN25_7B_INSTRUCT, QWEN3_8B, QWEN3_30B_A3B,
                                TINY_QWEN2, TINY_QWEN2_D128, TINY_QWEN3, TINY_QWEN3_MOE, TINY_QWEN3_MOE_UNNORM)}


MOE_MAX_EXPERTS, MOE_MAX_TOP_K = 256, 16


def check_moe(cfg: ShardModelConfig) -> None:
    """Raise NotImplementedError for a MoE config the kernels (csrc/moe.cu) cannot take."""
    if not cfg.is_moe:
        return
    E, k, H, Ie = cfg.n_experts, cfg.top_k, cfg.hidden, cfg.moe_intermediate
    if not (E <= MOE_MAX_EXPERTS and 1 <= k <= min(MOE_MAX_TOP_K, E)):
        raise NotImplementedError(f"{cfg.name}: {E} experts, {k} per token: the MoE kernels take at most "
                                  f"{MOE_MAX_EXPERTS} experts and 1 <= top_k <= min({MOE_MAX_TOP_K}, experts)")
    if H % 128 or Ie % 64 or H * 2 > 48 * 1024 or k * Ie * 2 > 48 * 1024:
        raise NotImplementedError(f"{cfg.name}: hidden {H} / moe_intermediate {Ie}: the MoE kernels need hidden % 128 == 0, "
                                  f"moe_intermediate % 64 == 0, hidden <= 24576 and top_k * moe_intermediate <= 24576")


def moe_fields(model_type: str, get) -> dict:
    """The MoE fields of ShardModelConfig from an HF config (``get(key)`` reads one of its values): {} for a dense
    qwen2 / qwen3 model.  Qwen3-MoE runs when every layer is sparse; other MoE families raise NotImplementedError."""
    if model_type != "qwen3_moe":
        # any other config that names routed experts (Mixtral, Qwen2-MoE, DeepSeek, DBRX, ...) is a MoE family too
        if "moe" in model_type or any(get(k) for k in ("num_experts", "num_local_experts", "n_routed_experts",
                                                        "moe_num_experts", "ffn_config")):
            raise NotImplementedError(f"model_type {model_type!r}: of the mixture-of-experts families only qwen3_moe runs "
                                      "here (no shared expert)")
        return {}
    if get("mlp_only_layers") or int(get("decoder_sparse_step") or 1) != 1:
        raise NotImplementedError("qwen3_moe with mixed dense and sparse layers (mlp_only_layers / decoder_sparse_step != 1)")
    if get("output_router_logits"):
        raise NotImplementedError("output_router_logits=True: router logits are not returned")
    # transformers 5 writes the expert count as num_local_experts (num_experts is its attribute alias)
    E = get("num_experts") if get("num_experts") is not None else get("num_local_experts")
    return dict(n_experts=int(E), top_k=int(get("num_experts_per_tok")),
                moe_intermediate=int(get("moe_intermediate_size")), norm_topk_prob=bool(get("norm_topk_prob")))


def get_config(name: str) -> ShardModelConfig:
    try:
        return REGISTRY[name]
    except KeyError as e:
        raise KeyError(f"unknown model {name!r}; known: {sorted(REGISTRY)}") from e
