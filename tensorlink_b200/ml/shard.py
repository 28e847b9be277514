"""The CUDA shard operator: a contiguous layer range executed by the sm_90a kernels.

Mirrors the reference's shard operator ``LayerGroupModule`` (/root/reference/tensorlink/ml/injector.py:154-281):
same constructor role (a list of layers + the loop live-ins), ``num_layers`` attribute, ``forward(**kwargs) ->
dict`` returning ``kwargs ∪ {hidden_states}``.  What differs is everything underneath: instead of ``exec``-ing
HF's loop body over ``nn.Module`` layers, each layer is five to eight kernel launches on a resident bf16
parameter arena with a resident KV cache; masks, RoPE tables and positions are generated on the device and
never cross a shard boundary (the reference ships them with every call, injector.py:508-556).

HBM layout (per shard):
  params   one flat bf16 arena; per layer  ln1 | wqkv[(n_h+2n_kv)d, H] | bqkv | (q_norm,k_norm) | wo[H, n_h d] |
           ln2 | wgu[2I, H] (row 2j = gate_j, row 2j+1 = up_j) | wd[H, I]; then embed / final norm / lm_head
           on the ranks that own them.  Every tensor starts on a 256-byte boundary (TMA needs 16).
  fp8      FP8 shards (``ShardParams(fp8=True)``, ml/fp8.py): the four Linear weights of every layer live instead in a
           float8_e4m3fn arena in the same row layout (256-byte boundaries), with fp32 scales [N, K/128] per row in a
           third arena; norms, biases, embed, final norm and lm_head stay in the bf16 arena.
  kv       per layer K and V  [B_max, n_kv, T_max, d] bf16 (head-major: decode streams [T, d] per head).
  act      x[N,H], qkv[N,(n_h+2n_kv)d], q[N,n_h d], attn[N,n_h d], h[N,H], act[N,I]  for N = B*S tokens.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence

import torch

from .. import native as nat
from . import fp8 as F8
from .configs import ShardModelConfig, check_moe
from .weights import init_state_dict

ALIGN = 128  # elements (256 B)


_GEMV_MAX_ROWS = None


def gemv_max_rows() -> int:
    """Rows per decode step up to which the weight-streaming GEMV path is used; more rows go through the wgmma GEMM
    path (one weight pass for all rows; the GEMV kernel needs a second pass above 4 rows and spends CUDA-core FMAs per
    row).  Default 3, not yet re-chosen by measurement on H100; TL_GEMV_MAX_ROWS overrides (1..8)."""
    global _GEMV_MAX_ROWS
    if _GEMV_MAX_ROWS is None:
        import os
        _GEMV_MAX_ROWS = max(1, min(8, int(os.environ.get("TL_GEMV_MAX_ROWS", "3"))))
    return _GEMV_MAX_ROWS


_FP8_GEMV_MAX_ROWS = None


def fp8_gemv_max_rows() -> int:
    """``gemv_max_rows()`` for FP8 shards: rows per step up to which the FP8 weight-streaming GEMV runs (in passes of at
    most 4 rows, one byte per weight each); more rows dequantize each Linear into a bf16 scratch buffer and run the GEMM
    path (about 5 bytes per weight).  Default 4, one GEMV pass: measured on an H100 SXM (700 W) with tools/bench_fp8.py,
    the GEMV wins at 4 rows for Qwen2.5-7B and Qwen3-8B, while at 6..8 rows (two passes) the two models disagree
    (DESIGN.md §4.1).  TL_FP8_GEMV_MAX_ROWS overrides (1..8)."""
    global _FP8_GEMV_MAX_ROWS
    if _FP8_GEMV_MAX_ROWS is None:
        import os
        _FP8_GEMV_MAX_ROWS = max(1, min(8, int(os.environ.get("TL_FP8_GEMV_MAX_ROWS", "4"))))
    return _FP8_GEMV_MAX_ROWS


def fp8_gemv_rows(cfg: ShardModelConfig) -> int:
    """Rows per step up to which an FP8 stage of ``cfg`` runs the FP8 GEMV: ``fp8_gemv_max_rows()``, lowered so that
    one pass (at most 4 rows) of staged activations fits the register-streaming kernel's shared memory for the widest
    Linear input (the down projection's K = intermediate).  That kernel is where a pass goes when x leaves the
    weight-streaming ring too few stages, as for the bf16 GEMV; past it the step takes the dequantize + GEMM path."""
    K = max(cfg.hidden, cfg.q_dim, cfg.intermediate)
    fit = 0
    while fit < 4 and (fit + 1) * K * 2 + 256 * (fit + 1) <= 200 * 1024:       # x rows + the epilogue's partial sums
        fit += 1
    return min(fp8_gemv_max_rows(), fit)


def _rope_inv_freq(cfg: ShardModelConfig) -> torch.Tensor:
    """site-packages/transformers/models/qwen2/modeling_qwen2.py:84-99, computed on the host in fp32 like HF."""
    d = cfg.head_dim
    return 1.0 / (cfg.rope_theta ** (torch.arange(0, d, 2, dtype=torch.int64).to(torch.float32) / d))


class ShardParams:
    """Flat bf16 parameter arena of one shard, with fused-QKV / interleaved gate-up views.  ``fp8=True``: the decoder
    layers' Linear weights are float8_e4m3fn views (``v``) with per-row scales (``s``), see the module docstring."""

    def __init__(self, cfg: ShardModelConfig, layer_ids: Sequence[int], has_embed: bool, has_head: bool,
                 device, with_grad: bool = False, fp8: bool = False):
        if fp8 and with_grad:
            raise NotImplementedError("training with FP8 weights is not supported (load the model with training=False)")
        check_moe(cfg)
        if cfg.is_moe and (fp8 or with_grad):
            raise NotImplementedError("a Qwen3-MoE model runs bf16 inference only: " +
                                      ("FP8 MoE weights are not supported" if fp8 else "training is not supported"))
        self.fp8 = bool(fp8)
        self.cfg, self.layer_ids = cfg, list(layer_ids)
        self.has_embed, self.has_head = has_embed, has_head
        self.device = torch.device(device)
        H, I = cfg.hidden, cfg.intermediate
        spec: List[tuple] = []
        for li in self.layer_ids:
            spec += [(f"l{li}.ln1", (H,)), (f"l{li}.wqkv", (cfg.qkv_dim, H))]
            if cfg.qkv_bias:
                spec.append((f"l{li}.bqkv", (cfg.qkv_dim,)))
            if cfg.qk_norm:
                spec += [(f"l{li}.qn", (cfg.head_dim,)), (f"l{li}.kn", (cfg.head_dim,))]
            spec += [(f"l{li}.wo", (H, cfg.q_dim)), (f"l{li}.ln2", (H,))]
            if cfg.is_moe:
                E, Ie = cfg.n_experts, cfg.moe_intermediate
                spec += [(f"l{li}.router", (E, H)), (f"l{li}.ewgu", (E, 2 * Ie, H)), (f"l{li}.ewd", (E, H, Ie))]
            else:
                spec += [(f"l{li}.wgu", (2 * I, H)), (f"l{li}.wd", (H, I))]
        if has_embed:
            spec.append(("embed", (cfg.vocab, H)))
        if has_head:
            spec.append(("norm", (H,)))
            if not (cfg.tied and has_embed):
                spec.append(("head", (cfg.vocab, H)))
        qspec = [(n, sh) for n, sh in spec if n.split(".")[-1] in F8.LINEARS] if self.fp8 else []
        spec = [(n, sh) for n, sh in spec if (n, sh) not in qspec]
        self.spec = spec
        self.offsets: Dict[str, tuple] = {}
        off = 0
        for name, shape in spec:
            n = 1
            for s in shape:
                n *= s
            self.offsets[name] = (off, n, shape)
            off += (n + ALIGN - 1) // ALIGN * ALIGN
        self.numel = off
        self.flat = torch.zeros(off, dtype=torch.bfloat16, device=self.device)
        self.grad: Optional[torch.Tensor] = torch.zeros_like(self.flat) if with_grad else None
        self.v: Dict[str, torch.Tensor] = {n: self.flat[o:o + k].view(shape) for n, (o, k, shape) in self.offsets.items()}
        self.g: Dict[str, torch.Tensor] = ({n: self.grad[o:o + k].view(shape) for n, (o, k, shape) in self.offsets.items()}
                                           if with_grad else {})
        if has_head and cfg.tied and has_embed:
            self.v["head"] = self.v["embed"]
            if with_grad:
                self.g["head"] = self.g["embed"]
        self.s: Dict[str, torch.Tensor] = {}
        self.q8 = self.scales = self.deq = None
        if qspec:
            qoff, soff, at = 0, 0, {}
            for name, (N, K) in qspec:
                at[name] = (qoff, soff, N, K)
                qoff += (N * K + 255) // 256 * 256
                soff += (N * (K // F8.BLOCK) + 63) // 64 * 64
            self.q8 = torch.zeros(qoff, dtype=torch.float8_e4m3fn, device=self.device)
            self.scales = torch.zeros(soff, dtype=torch.float32, device=self.device)
            for name, (qo, so, N, K) in at.items():
                self.v[name] = self.q8[qo:qo + N * K].view(N, K)
                self.s[name] = self.scales[so:so + N * (K // F8.BLOCK)].view(N, K // F8.BLOCK)
            # the GEMM paths' bf16 copy of one Linear at a time (dequant_fp8), sized for the largest
            self.deq = torch.empty(max(N * K for _, (N, K) in qspec), dtype=torch.bfloat16, device=self.device)

    # ---- HF state dict  <->  fused layout ------------------------------------------------------------
    def load_hf_state_dict(self, sd: Dict[str, torch.Tensor]):
        """Fuse q/k/v, interleave gate/up (the role of worker.py:542-638 ``_load_grouped_layer_weights``)."""
        cfg = self.cfg
        dev = self.device

        def put(name, t):
            self.v[name].copy_(t.to(device=dev, dtype=torch.bfloat16))

        for li in self.layer_ids:
            p = f"model.layers.{li}."
            put(f"l{li}.ln1", sd[p + "input_layernorm.weight"])
            if self.fp8:
                self._load_linears_fp8(sd, li)
            else:
                put(f"l{li}.wqkv", torch.cat([sd[p + "self_attn.q_proj.weight"], sd[p + "self_attn.k_proj.weight"],
                                              sd[p + "self_attn.v_proj.weight"]], dim=0))
            if cfg.qkv_bias:
                put(f"l{li}.bqkv", torch.cat([sd[p + "self_attn.q_proj.bias"], sd[p + "self_attn.k_proj.bias"],
                                              sd[p + "self_attn.v_proj.bias"]], dim=0))
            if cfg.qk_norm:
                put(f"l{li}.qn", sd[p + "self_attn.q_norm.weight"])
                put(f"l{li}.kn", sd[p + "self_attn.k_norm.weight"])
            put(f"l{li}.ln2", sd[p + "post_attention_layernorm.weight"])
            if cfg.is_moe:
                put(f"l{li}.wo", sd[p + "self_attn.o_proj.weight"])
                self._load_experts(sd, li)
            elif not self.fp8:
                put(f"l{li}.wo", sd[p + "self_attn.o_proj.weight"])
                g, u = sd[p + "mlp.gate_proj.weight"], sd[p + "mlp.up_proj.weight"]
                put(f"l{li}.wgu", torch.stack([g, u], dim=1).reshape(2 * cfg.intermediate, cfg.hidden))
                put(f"l{li}.wd", sd[p + "mlp.down_proj.weight"])
        if self.has_embed:
            put("embed", sd["model.embed_tokens.weight"])
        if self.has_head:
            put("norm", sd["model.norm.weight"])
            if not (cfg.tied and self.has_embed):
                put("head", sd["lm_head.weight"] if "lm_head.weight" in sd else sd["model.embed_tokens.weight"])

    def hf_state_dict(self, grads: bool = False) -> Dict[str, torch.Tensor]:
        """Inverse mapping (the role of ``parameters(distributed=True)``, module.py:577-650).  An FP8 shard returns HF's
        quantized names: ``...weight`` as float8_e4m3fn and ``...weight_scale_inv`` as the fp32 [N/128, K/128] grid."""
        cfg = self.cfg
        if grads and getattr(self, "grad_settle", None) is not None:
            self.grad_settle()          # matrix gradients are zeroed lazily after zero_grad() (ml/train.py)
        src = self.g if grads else self.v
        out: Dict[str, torch.Tensor] = {}
        for li in self.layer_ids:
            p = f"model.layers.{li}."
            out[p + "input_layernorm.weight"] = src[f"l{li}.ln1"].clone()
            q, k, v = src[f"l{li}.wqkv"].split([cfg.q_dim, cfg.kv_dim, cfg.kv_dim], dim=0)
            out[p + "self_attn.q_proj.weight"], out[p + "self_attn.k_proj.weight"] = q.clone(), k.clone()
            out[p + "self_attn.v_proj.weight"] = v.clone()
            if cfg.qkv_bias:
                bq, bk, bv = src[f"l{li}.bqkv"].split([cfg.q_dim, cfg.kv_dim, cfg.kv_dim], dim=0)
                out[p + "self_attn.q_proj.bias"], out[p + "self_attn.k_proj.bias"] = bq.clone(), bk.clone()
                out[p + "self_attn.v_proj.bias"] = bv.clone()
            if cfg.qk_norm:
                out[p + "self_attn.q_norm.weight"] = src[f"l{li}.qn"].clone()
                out[p + "self_attn.k_norm.weight"] = src[f"l{li}.kn"].clone()
            out[p + "self_attn.o_proj.weight"] = src[f"l{li}.wo"].clone()
            out[p + "post_attention_layernorm.weight"] = src[f"l{li}.ln2"].clone()
            if cfg.is_moe:
                E, Ie, H = cfg.n_experts, cfg.moe_intermediate, cfg.hidden
                gu = src[f"l{li}.ewgu"].view(E, Ie, 2, H)
                out[p + "mlp.gate.weight"] = src[f"l{li}.router"].clone()
                out[p + "mlp.experts.gate_up_proj"] = torch.cat([gu[:, :, 0], gu[:, :, 1]], dim=1)
                out[p + "mlp.experts.down_proj"] = src[f"l{li}.ewd"].clone()
                continue
            gu = src[f"l{li}.wgu"].view(cfg.intermediate, 2, cfg.hidden)
            out[p + "mlp.gate_proj.weight"], out[p + "mlp.up_proj.weight"] = gu[:, 0].clone(), gu[:, 1].clone()
            out[p + "mlp.down_proj.weight"] = src[f"l{li}.wd"].clone()
        if self.has_embed:
            out["model.embed_tokens.weight"] = src["embed"].clone()
        if self.has_head:
            out["model.norm.weight"] = src["norm"].clone()
            # tied heads appear under both names, like HF's own state_dict()
            out["lm_head.weight"] = out["model.embed_tokens.weight"] if (cfg.tied and self.has_embed) else src["head"].clone()
        return self._with_scale_grids(out) if self.fp8 else out

    def _load_experts(self, sd, li: int):
        """Layer li's router and experts, from HF's fused in-memory names (``mlp.experts.gate_up_proj`` [E, 2I, H] with
        the gate rows first, ``mlp.experts.down_proj`` [E, H, I]) or the checkpoints' per-expert names
        (``mlp.experts.{e}.{gate,up,down}_proj.weight``).  Gate/up rows are interleaved per expert as in ``wgu``."""
        cfg, p = self.cfg, f"model.layers.{li}."
        E, Ie, H = cfg.n_experts, cfg.moe_intermediate, cfg.hidden
        dev = self.device
        self.v[f"l{li}.router"].copy_(sd[p + "mlp.gate.weight"].to(device=dev, dtype=torch.bfloat16))
        gu, dn = self.v[f"l{li}.ewgu"].view(E, Ie, 2, H), self.v[f"l{li}.ewd"]
        if p + "mlp.experts.gate_up_proj" in sd:
            w = sd[p + "mlp.experts.gate_up_proj"].to(device=dev, dtype=torch.bfloat16)
            gu[:, :, 0].copy_(w[:, :Ie])
            gu[:, :, 1].copy_(w[:, Ie:])
            dn.copy_(sd[p + "mlp.experts.down_proj"].to(device=dev, dtype=torch.bfloat16))
            return
        for e in range(E):
            q = f"{p}mlp.experts.{e}."
            gu[e, :, 0].copy_(sd[q + "gate_proj.weight"].to(device=dev, dtype=torch.bfloat16))
            gu[e, :, 1].copy_(sd[q + "up_proj.weight"].to(device=dev, dtype=torch.bfloat16))
            dn[e].copy_(sd[q + "down_proj.weight"].to(device=dev, dtype=torch.bfloat16))

    def _load_linears_fp8(self, sd, li: int):
        """Layer li's four Linears from HF's FP8 weight + scale_inv grid of each projection (a bf16 weight is quantized
        first, by HF's rule), fused like the bf16 arena: q/k/v concatenated, gate/up row-interleaved."""
        p = f"model.layers.{li}."
        for name, projs in (("wqkv", ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj")),
                            ("wo", ("self_attn.o_proj",)), ("wgu", ("mlp.gate_proj", "mlp.up_proj")),
                            ("wd", ("mlp.down_proj",))):
            qs, rs = [], []
            for pre in (p + j for j in projs):
                w = sd[pre + ".weight"]
                if w.dtype == torch.float8_e4m3fn:
                    q, inv = w.to(self.device), sd[pre + ".weight_scale_inv"].to(self.device)
                else:
                    q, inv = F8.quantize(w.to(self.device))
                if tuple(inv.shape) != (q.shape[0] // F8.BLOCK, q.shape[1] // F8.BLOCK):
                    raise NotImplementedError(f"{pre}.weight_scale_inv of shape {tuple(inv.shape)} for a weight of "
                                              f"{tuple(q.shape)}: only 128x128 blocks are supported")
                qs.append(q)
                rs.append(F8.rows_from_grid(inv))
            cat = (lambda ts: torch.stack(ts, dim=1).flatten(0, 1)) if name == "wgu" else (lambda ts: torch.cat(ts, dim=0))
            self.v[f"l{li}.{name}"].copy_(cat(qs))
            self.s[f"l{li}.{name}"].copy_(cat(rs))

    def _with_scale_grids(self, out: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        """``out`` with each FP8 ``...weight`` followed by its ``...weight_scale_inv`` grid, recovered from the rows."""
        cfg, grids = self.cfg, {}
        for li in self.layer_ids:
            p = f"model.layers.{li}."
            for pre, r in zip(("q_proj", "k_proj", "v_proj"),
                              self.s[f"l{li}.wqkv"].split([cfg.q_dim, cfg.kv_dim, cfg.kv_dim], dim=0)):
                grids[p + "self_attn." + pre] = r
            grids[p + "self_attn.o_proj"] = self.s[f"l{li}.wo"]
            sgu = self.s[f"l{li}.wgu"].view(cfg.intermediate, 2, -1)
            grids[p + "mlp.gate_proj"], grids[p + "mlp.up_proj"] = sgu[:, 0], sgu[:, 1]
            grids[p + "mlp.down_proj"] = self.s[f"l{li}.wd"]
        res: Dict[str, torch.Tensor] = {}
        for k, t in out.items():
            res[k] = t
            pre = k[:-len(".weight")]
            if k.endswith(".weight") and pre in grids:
                res[pre + ".weight_scale_inv"] = F8.grid_from_rows(grids[pre])
        return res

    def init_seeded(self, seed: int = 1234):
        """Same values the CPU oracle draws (weights.init_state_dict), materialised layer by layer."""
        cfg = self.cfg
        for li in self.layer_ids:
            sd = init_state_dict(cfg, seed, torch.bfloat16, "cpu", layers=[li], with_embed=False, with_head=False)
            sub = ShardParams.__new__(ShardParams)
            sub.__dict__.update(self.__dict__)
            sub.layer_ids, sub.has_embed, sub.has_head = [li], False, False
            sub.load_hf_state_dict(sd)
        sd = init_state_dict(cfg, seed, torch.bfloat16, "cpu", layers=[], with_embed=self.has_embed or (
            self.has_head and cfg.tied), with_head=self.has_head)
        sub = ShardParams.__new__(ShardParams)
        sub.__dict__.update(self.__dict__)
        sub.layer_ids = []
        sub.load_hf_state_dict(sd)

    def init_on_device(self, seed: int = 1234, std: float = 0.02):
        """Random init drawn directly on the GPU (benchmarks at 7B/8B scale; not comparable with the oracle).  An FP8
        shard draws each Linear's bf16 projections the same way and quantizes them on the device."""
        g = torch.Generator(device=self.device).manual_seed(seed)
        self.flat.normal_(0.0, std, generator=g)
        for name in self.v:
            if name.endswith(("ln1", "ln2", "qn", "kn")) or name == "norm":
                self.v[name].fill_(1.0)
        if self.fp8:
            cfg, H, I = self.cfg, self.cfg.hidden, self.cfg.intermediate
            shapes = {"self_attn.q_proj": (cfg.q_dim, H), "self_attn.k_proj": (cfg.kv_dim, H),
                      "self_attn.v_proj": (cfg.kv_dim, H), "self_attn.o_proj": (H, cfg.q_dim), "mlp.gate_proj": (I, H),
                      "mlp.up_proj": (I, H), "mlp.down_proj": (H, I)}
            for li in self.layer_ids:
                sd = {f"model.layers.{li}.{k}.weight": torch.empty(shape, dtype=torch.bfloat16, device=self.device).normal_(
                    0.0, std, generator=g) for k, shape in shapes.items()}
                self._load_linears_fp8(sd, li)


@dataclass
class ShardBuffers:
    """Activation workspaces for up to ``n_max`` tokens in flight."""
    x: torch.Tensor
    h: torch.Tensor
    qkv: torch.Tensor
    q: torch.Tensor
    attn: torch.Tensor
    act: torch.Tensor
    moe: Optional["MoeBuffers"] = None        # routing buffers of a MoE stage


class MoeBuffers:
    """Routing buffers of a Qwen3-MoE stage for up to ``n`` tokens: router logits, the picks and their weights, the
    grouped-GEMM plan (csrc/moe.cu) and the gathered rows; decode rows use ``act[:n*k]`` for their expert activations."""

    def __init__(self, cfg: ShardModelConfig, n: int, device):
        E, k, H, Ie = cfg.n_experts, cfg.top_k, cfg.hidden, cfg.moe_intermediate
        i32 = dict(dtype=torch.int32, device=device)
        self.n, self.tiles_max = n, nat.moe_max_tiles(n, E, k)
        rows = self.tiles_max * 128
        self.logits = torch.empty(n, E, dtype=torch.bfloat16, device=device)
        self.ids, self.wts = torch.empty(n, k, **i32), torch.empty(n, k, dtype=torch.float32, device=device)
        self.counts, self.offsets, self.row_of = torch.empty(E, **i32), torch.empty(E + 1, **i32), torch.empty(n * k, **i32)
        self.tiles = torch.empty(self.tiles_max, 2, **i32)
        self.hg = torch.empty(rows, H, dtype=torch.bfloat16, device=device)
        self.act = torch.empty(rows, Ie, dtype=torch.bfloat16, device=device)
        self.y = torch.empty(rows, H, dtype=torch.bfloat16, device=device)


class CudaLayerGroup:
    """CUDA shard operator (LayerGroupModule mirror, injector.py:154-281)."""

    def __init__(self, cfg: ShardModelConfig, params: ShardParams, max_batch: int, max_seq: int,
                 max_tokens: Optional[int] = None):
        nat.require_device()
        self.cfg, self.p = cfg, params
        self.layer_ids = params.layer_ids
        self.num_layers = len(self.layer_ids)             # worker.py:332-335 dispatches on this attribute
        self.input_vars = ["hidden_states", "past_len", "use_cache"]
        self.output_vars = ["hidden_states"]
        self.device = params.device
        self.B_max, self.T_max = max_batch, max_seq
        dev, bf = self.device, torch.bfloat16
        self.kc = [torch.zeros(max_batch, cfg.n_kv_heads, max_seq, cfg.head_dim, dtype=bf, device=dev)
                   for _ in self.layer_ids]
        self.vc = [torch.zeros_like(k) for k in self.kc]
        self.cos, self.sin = nat.rope_table(_rope_inv_freq(cfg).to(dev), max_seq)
        # what the launch after this shard's last decode GEMV streams (a prefetch hint only, see _layer_decode)
        self.weights_after_last_layer = (params.v.get("head") if "head" in params.v else
                                         params.v.get(f"l{self.layer_ids[0]}.wqkv") if len(self.layer_ids) else None)
        self.pos_dev = torch.zeros(1, dtype=torch.int32, device=dev)      # next write position in the cache
        self.kvlen_dev = torch.zeros(1, dtype=torch.int32, device=dev)    # valid keys for the decode kernel
        # left-padded rows: kv_start[b] leading cache slots of row b are pad (never attended; RoPE position = slot -
        # kv_start[b]).  Set by prefill(kv_start=...), constant through the decode steps that follow it.
        self.kv_start_dev = torch.zeros(max_batch, dtype=torch.int32, device=dev)
        self.ragged = False
        self.n_max = max_tokens or max_batch * max_seq
        self._alloc_bufs(min(self.n_max, 8))
        self.dbufs = self._make_bufs(max_batch)       # decode-time buffers: fixed addresses (captured graphs, job lists)
        self.moe_pf: Optional[MoeBuffers] = None
        if cfg.is_moe:
            self.dbufs.moe = MoeBuffers(cfg, max_batch, dev)
        # ticket counters of the four decode GEMVs of every layer (_layer_decode): one block per call site, so no two
        # launches that can overlap share one, and captured graphs keep fixed addresses
        self.gemv_ctr = nat.gemv_counters(self.num_layers, 4, device=dev)
        # split-K workspace for batched decode (rows above the GEMV threshold, <= 128): the qkv / o / down Linears have
        # too few output tiles to occupy every SM
        self.gemm_ws = (torch.empty(nat.gemm_splitk_ws(min(max_batch, 128), max(cfg.qkv_dim, cfg.hidden)), dtype=torch.uint8,
                                    device=dev) if max_batch > 1 else None)
        self.dec_ws = torch.empty(max(nat.attn_decode_ws(max_batch, cfg.n_heads, cfg.head_dim, max_seq), 16),
                                  dtype=torch.uint8, device=dev)
        self.scale = cfg.head_dim ** -0.5
        self.vbufs: Optional[ShardBuffers] = None     # verify step (verify_step_inplace): its own buffers, on first use
        self.ver_gemm_ws = self.ver_attn_ws = None
        self.allow_chain = True              # DistributedModel clears it when NCCL kernels share the device during decode
        self.chain_sync: Optional[torch.Tensor] = None
        self.chain_attn_ws: Optional[torch.Tensor] = None
        self._chains: Dict[tuple, list] = {}

    def _make_bufs(self, n: int) -> ShardBuffers:
        cfg, dev, bf = self.cfg, self.device, torch.bfloat16
        return ShardBuffers(
            x=torch.empty(n, cfg.hidden, dtype=bf, device=dev), h=torch.empty(n, cfg.hidden, dtype=bf, device=dev),
            qkv=torch.empty(n, cfg.qkv_dim, dtype=bf, device=dev), q=torch.empty(n, cfg.q_dim, dtype=bf, device=dev),
            attn=torch.empty(n, cfg.q_dim, dtype=bf, device=dev),
            act=torch.empty(n, cfg.intermediate, dtype=bf, device=dev))

    def _alloc_bufs(self, n: int):
        self.bufs = self._make_bufs(n)
        self.n_alloc = n

    def _dbufs(self, n: int) -> ShardBuffers:
        b = self.dbufs
        return ShardBuffers(b.x[:n], b.h[:n], b.qkv[:n], b.q[:n], b.attn[:n], b.act[:n], b.moe)

    def _bufs(self, n: int) -> ShardBuffers:
        if n > self.n_alloc:
            self._alloc_bufs(n)
        b = self.bufs
        if self.cfg.is_moe and (self.moe_pf is None or self.moe_pf.n < n):
            self.moe_pf = MoeBuffers(self.cfg, n, self.device)
        return ShardBuffers(b.x[:n], b.h[:n], b.qkv[:n], b.q[:n], b.attn[:n], b.act[:n], self.moe_pf)

    # ------------------------------------------------------------------------------------------ cache control
    def reset_cache(self, past_len: int = 0):
        self.pos_dev.fill_(past_len)
        self.kvlen_dev.fill_(past_len)

    # ------------------------------------------------------------------------------------------ layer bodies
    def _gemv(self, x: torch.Tensor, name: str, **kw) -> torch.Tensor:
        """The decode Linear ``name`` of the arena: the bf16 GEMV, or on an FP8 shard the FP8 GEMV over its scales."""
        p = self.p
        if p.fp8:
            return nat.gemv_fp8(x, p.v[name], p.s[name], **kw)
        return nat.gemv(x, p.v[name], **kw)

    def _gemm(self, a: torch.Tensor, name: str, **kw) -> torch.Tensor:
        """The GEMM Linear ``name``; an FP8 shard first dequantizes it into the shard's bf16 scratch (one Linear at a
        time: the launches run in stream order)."""
        p = self.p
        w = nat.dequant_fp8(p.v[name], p.s[name], out=p.deq) if p.fp8 else p.v[name]
        return nat.gemm(a, w, **kw)

    def gemv_rows(self) -> int:
        """Rows per step up to which decode and verify steps run the weight-streaming GEMVs."""
        return fp8_gemv_rows(self.cfg) if self.p.fp8 else gemv_max_rows()

    def _kv_start(self):
        """The per-row key starts for the attention and RoPE launches, or None (every row starts at slot 0)."""
        return self.kv_start_dev if self.ragged else None

    def _layer_prefill(self, j: int, x: torch.Tensor, B: int, S: int, past_len: int, w: ShardBuffers):
        """site-packages/transformers/models/qwen2/modeling_qwen2.py:280-310 for N = B*S tokens (GEMM path)."""
        cfg, v, li = self.cfg, self.p.v, self.layer_ids[j]
        ks = self._kv_start()
        nat.rmsnorm_fwd(x, v[f"l{li}.ln1"], cfg.rms_eps, out=w.h)
        self._gemm(w.h, f"l{li}.wqkv", out=w.qkv, bias=v.get(f"l{li}.bqkv"))
        nat.rope_kv_fwd(w.qkv, w.q, self.kc[j], self.vc[j], self.pos_dev, self.cos, self.sin, v.get(f"l{li}.qn"),
                        v.get(f"l{li}.kn"), cfg.rms_eps, S, cfg.n_heads, cfg.n_kv_heads, cfg.head_dim, kv_start=ks)
        nat.attn_prefill_fwd(w.q, self.kc[j], self.vc[j], w.attn, None, B, S, past_len, cfg.n_heads, cfg.n_kv_heads,
                             cfg.head_dim, self.scale, kv_start=ks)
        self._gemm(w.attn, f"l{li}.wo", out=x, residual=x)
        nat.rmsnorm_fwd(x, v[f"l{li}.ln2"], cfg.rms_eps, out=w.h)
        if cfg.is_moe:
            self._moe_grouped(li, x, w.h, w.moe)
            return
        self._gemm(w.h, f"l{li}.wgu", out=w.act, flags=nat.EPI_SWIGLU)
        self._gemm(w.act, f"l{li}.wd", out=x, residual=x)

    def _moe_grouped(self, li: int, x: torch.Tensor, h: torch.Tensor, mb: MoeBuffers, out: Optional[torch.Tensor] = None):
        """Qwen3-MoE block for the N rows of ``h`` (the normed ``x``): router GEMM -> route + plan -> gather -> grouped
        gate/up (SwiGLU) -> grouped down -> combine, out = bf16(x + acc) (into ``x`` unless ``out``)."""
        cfg, v = self.cfg, self.p.v
        n, k = h.shape[0], cfg.top_k
        T = nat.moe_max_tiles(n, cfg.n_experts, k)
        nat.gemm(h, v[f"l{li}.router"], out=mb.logits[:n])
        row_of, tiles = mb.row_of[:n * k], mb.tiles[:T]
        nat.moe_route(mb.logits[:n], k, cfg.norm_topk_prob, mb.ids[:n], mb.wts[:n], (mb.counts, mb.offsets, row_of, tiles))
        nat.moe_gather(h, row_of, mb.hg[:T * 128], k)
        nat.moe_gemm(mb.hg[:T * 128], v[f"l{li}.ewgu"], mb.act[:T * 128], tiles, flags=nat.EPI_SWIGLU)
        nat.moe_gemm(mb.act[:T * 128], v[f"l{li}.ewd"], mb.y[:T * 128], tiles)
        nat.moe_combine(mb.y[:T * 128], row_of, mb.wts[:n], x, x if out is None else out)

    def _layer_decode_moe(self, j: int, x: torch.Tensor, B: int, w: ShardBuffers, out: Optional[torch.Tensor], attention):
        """``_layer_decode`` of a MoE layer: the attention half as in the dense layer, then norm -> router GEMV -> route ->
        expert GEMV gate/up over the picked experts only -> expert GEMV down with the combine and the residual."""
        cfg, v, li, mb = self.cfg, self.p.v, self.layer_ids[j], w.moe
        ctr = self.gemv_ctr[j]
        self._gemv(x, f"l{li}.wqkv", out=w.qkv, bias=v.get(f"l{li}.bqkv"), norm_w=v[f"l{li}.ln1"], eps=cfg.rms_eps,
                   next_w=v[f"l{li}.wo"], counter=ctr[0])
        attention(j, li, B, w)
        self._gemv(w.attn, f"l{li}.wo", out=x, residual=x, next_w=v[f"l{li}.router"], counter=ctr[1])
        nat.rmsnorm_fwd(x, v[f"l{li}.ln2"], cfg.rms_eps, out=w.h)
        nat.gemv(w.h, v[f"l{li}.router"], out=mb.logits[:B], counter=ctr[2])
        nat.moe_route(mb.logits[:B], cfg.top_k, cfg.norm_topk_prob, mb.ids[:B], mb.wts[:B])
        act = mb.act[:B * cfg.top_k]
        nat.moe_gemv(w.h, v[f"l{li}.ewgu"], act, mb.ids[:B], flags=nat.EPI_SWIGLU)
        nat.moe_gemv(act, v[f"l{li}.ewd"], x if out is None else out, mb.ids[:B], wts=mb.wts[:B], residual=x,
                     flags=nat.EPI_RESIDUAL)

    FUSED_DECODE_MAX_T = 2048

    def _decode_attention(self, j: int, li: int, B: int, w: ShardBuffers):
        """w.qkv (post-bias) -> w.attn for one new token per row.  Short caches: one fused launch (RoPE + append +
        attention); long caches: RoPE/append, split-KV partials, reduce (three launches, parallel over the KV length)."""
        cfg, v = self.cfg, self.p.v
        ks = self._kv_start()
        if self.T_max <= self.FUSED_DECODE_MAX_T and (cfg.n_heads // cfg.n_kv_heads) <= 8:
            nat.attn_decode_fused(w.qkv, self.kc[j], self.vc[j], w.attn, self.pos_dev, self.cos, self.sin,
                                  v.get(f"l{li}.qn"), v.get(f"l{li}.kn"), cfg.rms_eps, B, cfg.n_heads, cfg.n_kv_heads,
                                  cfg.head_dim, self.scale, kv_start=ks)
            return
        nat.rope_kv_fwd(w.qkv, w.q, self.kc[j], self.vc[j], self.pos_dev, self.cos, self.sin, v.get(f"l{li}.qn"),
                        v.get(f"l{li}.kn"), cfg.rms_eps, 1, cfg.n_heads, cfg.n_kv_heads, cfg.head_dim, kv_start=ks)
        nat.attn_decode_fwd(w.q, self.kc[j], self.vc[j], w.attn, self.kvlen_dev, self.dec_ws, B, cfg.n_heads,
                            cfg.n_kv_heads, cfg.head_dim, self.scale, kv_start=ks)

    def _layer_decode(self, j: int, x: torch.Tensor, B: int, w: ShardBuffers, out: Optional[torch.Tensor] = None,
                      attention=None):
        """Same layer for B <= 8 single-token rows: weight-streaming GEMVs with the norms fused as prologues.
        ``attention``: what turns w.qkv into w.attn instead of ``_decode_attention`` (the verify step's)."""
        cfg, v, li = self.cfg, self.p.v, self.layer_ids[j]
        attention = attention or self._decode_attention
        if cfg.is_moe:
            return self._layer_decode_moe(j, x, B, w, out, attention)
        # every GEMV names the weights of the launch after it: it queues L2 prefetches behind its own loads, so HBM keeps
        # streaming through the launch boundary (and through the attention kernel) instead of idling there
        if j + 1 < self.num_layers:
            after = v[f"l{self.layer_ids[j + 1]}.wqkv"]
        else:
            after = self.weights_after_last_layer            # lm_head on the last stage, else layer 0 for the next slot
        ctr = self.gemv_ctr[j]
        self._gemv(x, f"l{li}.wqkv", out=w.qkv, bias=v.get(f"l{li}.bqkv"), norm_w=v[f"l{li}.ln1"], eps=cfg.rms_eps,
                   next_w=v[f"l{li}.wo"], counter=ctr[0])
        attention(j, li, B, w)
        self._gemv(w.attn, f"l{li}.wo", out=x, residual=x, next_w=v[f"l{li}.wgu"], counter=ctr[1])
        self._gemv(x, f"l{li}.wgu", out=w.act, norm_w=v[f"l{li}.ln2"], eps=cfg.rms_eps, flags=nat.EPI_SWIGLU,
                   next_w=v[f"l{li}.wd"], counter=ctr[2])
        self._gemv(w.act, f"l{li}.wd", out=x if out is None else out, residual=x, next_w=after, counter=ctr[3])

    def _layer_decode_batched(self, j: int, x: torch.Tensor, B: int, w: ShardBuffers, out: Optional[torch.Tensor] = None,
                              attention=None, ws: Optional[torch.Tensor] = None):
        """More single-token rows than the GEMV path takes: wgmma GEMMs in the weight-streaming regime (split along K
        where a Linear has too few output tiles to occupy every SM) + decode attention.  The RMSNorm after each
        residual Linear rides in that Linear's split-K reduce pass, so layer j > 0 finds its normalised input in w.h.
        ``attention`` / ``ws``: the verify step's attention and split-K workspace instead of the decode ones."""
        cfg, v, li = self.cfg, self.p.v, self.layer_ids[j]
        if ws is None:
            ws = self.gemm_ws if B <= 128 else None
        if cfg.is_moe:
            nat.rmsnorm_fwd(x, v[f"l{li}.ln1"], cfg.rms_eps, out=w.h)
            self._gemm(w.h, f"l{li}.wqkv", out=w.qkv, bias=v.get(f"l{li}.bqkv"), ws=ws)
            (attention or self._decode_attention)(j, li, B, w)
            self._gemm(w.attn, f"l{li}.wo", out=x, residual=x, ws=ws, norm_w=v[f"l{li}.ln2"], eps=cfg.rms_eps, h_out=w.h)
            self._moe_grouped(li, x, w.h, w.moe, out if j == self.num_layers - 1 else None)
            return
        if j == 0:
            nat.rmsnorm_fwd(x, v[f"l{li}.ln1"], cfg.rms_eps, out=w.h)
        self._gemm(w.h, f"l{li}.wqkv", out=w.qkv, bias=v.get(f"l{li}.bqkv"), ws=ws)
        (attention or self._decode_attention)(j, li, B, w)
        self._gemm(w.attn, f"l{li}.wo", out=x, residual=x, ws=ws, norm_w=v[f"l{li}.ln2"], eps=cfg.rms_eps, h_out=w.h)
        self._gemm(w.h, f"l{li}.wgu", out=w.act, flags=nat.EPI_SWIGLU, ws=ws)
        if j + 1 < self.num_layers:
            self._gemm(w.act, f"l{li}.wd", out=x, residual=x, ws=ws, norm_w=v[f"l{self.layer_ids[j + 1]}.ln1"],
                       eps=cfg.rms_eps, h_out=w.h)
        else:
            self._gemm(w.act, f"l{li}.wd", out=x if out is None else out, residual=x, ws=ws)

    def prefill(self, hidden: torch.Tensor, past_len: int = 0, kv_start=None) -> torch.Tensor:
        """hidden [B,S,H] -> [B,S,H]; appends S positions to the KV cache starting at ``past_len``.
        ``kv_start`` (B ints, or None): a left-padded batch, row b's first ``kv_start[b]`` cache slots being pad.  Those
        slots are never attended and row b's RoPE positions start at its first real token (HF's left-padded generation:
        position_ids = cumsum(mask) - 1).  The starts hold for the decode steps after this prefill, until the next one;
        the pad rows of the output are zero."""
        B, S, H = hidden.shape
        if B > self.B_max or past_len + S > self.T_max:
            raise ValueError(f"shard sized for B<={self.B_max}, T<={self.T_max}; got B={B}, T={past_len + S}")
        self._set_kv_start(kv_start, B, past_len + S)
        N = B * S
        w = self._bufs(N)
        w.x.copy_(hidden.reshape(N, H))
        self.pos_dev.fill_(past_len)
        for j in range(self.num_layers):
            self._layer_prefill(j, w.x, B, S, past_len, w)
        self.pos_dev.fill_(past_len + S)
        self.kvlen_dev.fill_(past_len + S)
        return w.x.view(B, S, H)

    def _set_kv_start(self, kv_start, B: int, T: int):
        if kv_start is None:
            self.ragged = False
            return
        ks = torch.as_tensor(kv_start, dtype=torch.int32).reshape(-1).cpu()
        if ks.numel() != B or bool((ks < 0).any()) or bool((ks >= T).any()):
            raise ValueError(f"kv_start needs {B} values in [0, {T}): every row keeps at least one real token")
        self.kv_start_dev.zero_()
        self.kv_start_dev[:B].copy_(ks, non_blocking=False)
        self.ragged = bool((ks != 0).any())

    def decode_step_inplace(self, x: torch.Tensor, out: Optional[torch.Tensor] = None, advance: bool = True):
        """x [B,H] updated in place through this shard's layers; one new token per row at position ``pos_dev``.
        Graph-capturable: the write position and the KV length live in device memory and are advanced by
        kernels inside the same launch sequence (kv_len += 1 before the layers, pos += 1 after).
        ``out``: where the LAST layer's down projection stores the shard's output rows instead of ``x`` — the next
        stage's peer-mapped input buffer (p2p/peer.py), so the hop rides on that kernel's own stores.
        ``advance=False``: the caller advances ``kvlen_dev`` before and ``pos_dev`` after (the mailbox kernels do)."""
        B = x.shape[0]
        w = self._dbufs(B)
        if advance:
            nat.advance_pos(self.kvlen_dev, None, 1)
        if self.chain_ok(B) or self.dq_ok(B):
            (self._decode_step_chained if self.chain_ok(B) else self._decode_step_dq)(x, B, out)
            if advance:
                nat.advance_pos(self.pos_dev, None, 1)
            return
        for j in range(self.num_layers):
            o = out if j == self.num_layers - 1 else None
            if B <= self.gemv_rows():
                self._layer_decode(j, x, B, w, o)
            else:
                self._layer_decode_batched(j, x, B, w, o)
        if advance:
            nat.advance_pos(self.pos_dev, None, 1)

    # ------------------------------------------------------------------------------------------ verify step
    def _verify_attention(self, j: int, li: int, n: int, w: ShardBuffers):
        """w.qkv (post-bias) of n consecutive tokens of cache row 0 -> w.attn: RoPE + append at pos..pos+n-1, then
        token i attends to keys 0..pos+i."""
        cfg, v = self.cfg, self.p.v
        nat.rope_kv_fwd(w.qkv, w.q, self.kc[j], self.vc[j], self.pos_dev, self.cos, self.sin, v.get(f"l{li}.qn"),
                        v.get(f"l{li}.kn"), cfg.rms_eps, n, cfg.n_heads, cfg.n_kv_heads, cfg.head_dim)
        nat.attn_verify_fwd(w.q, self.kc[j], self.vc[j], w.attn, self.pos_dev, self.ver_attn_ws, n, cfg.n_heads,
                            cfg.n_kv_heads, cfg.head_dim, self.scale)

    def verify_step_inplace(self, x: torch.Tensor):
        """x [n,H] (n <= 16): n consecutive tokens of cache row 0 at positions pos_dev.., updated in place through this
        shard's layers, as one graph-capturable launch sequence.  ``decode_step_inplace`` for n rows of one sequence:
        the same Linears (GEMVs up to gemv_max_rows(), else the split-K GEMMs), the per-kernel sequence always, and the
        verify attention.  Neither pos_dev nor kvlen_dev moves here (the accept step advances both).  The buffers are
        this step's own, at fixed addresses, allocated on first use; the GEMV ticket counters are the decode step's
        (each launch leaves its block zeroed, and a verify step never overlaps a decode step)."""
        n = x.shape[0]
        if not 1 <= n <= nat.VERIFY_MAX_ROWS:
            raise ValueError(f"verify step takes 1..{nat.VERIFY_MAX_ROWS} rows, got {n}")
        if self.ragged:
            raise NotImplementedError("verify step on a left-padded slot")
        if self.vbufs is None:
            cfg, dev, R = self.cfg, self.device, nat.VERIFY_MAX_ROWS
            self.vbufs = self._make_bufs(R)
            if cfg.is_moe:
                self.vbufs.moe = MoeBuffers(cfg, R, dev)
            self.ver_gemm_ws = torch.empty(nat.gemm_splitk_ws(R, max(cfg.qkv_dim, cfg.hidden)), dtype=torch.uint8, device=dev)
            self.ver_attn_ws = torch.empty(nat.attn_verify_ws(R, cfg.n_heads, cfg.head_dim, self.T_max), dtype=torch.uint8,
                                           device=dev)
        b = self.vbufs
        w = ShardBuffers(b.x[:n], b.h[:n], b.qkv[:n], b.q[:n], b.attn[:n], b.act[:n], b.moe)
        for j in range(self.num_layers):
            if n <= self.gemv_rows():
                self._layer_decode(j, x, n, w, attention=self._verify_attention)
            else:
                self._layer_decode_batched(j, x, n, w, attention=self._verify_attention, ws=self.ver_gemm_ws)

    # ------------------------------------------------------------------------------------------ chained decode step
    def chain_ok(self, B: int) -> bool:
        """Rows / shapes the persistent chain kernel (csrc/decode_chain.cu) takes.  Opt-in (TL_DECODE_IMPL=chain): it streams every Linear at
        the HBM rate but pays a software dependency (release/acquire counter + restaging the input vector) per phase where
        the default per-kernel sequence pays a programmatic-dependent-launch boundary."""
        import os
        cfg = self.cfg
        # the chain's ATTN job has no per-row key start: a left-padded slot takes the per-kernel sequence
        # the chain's GEMV jobs stream bf16 weights: an FP8 shard takes the per-kernel sequence
        return (os.environ.get("TL_DECODE_IMPL", "kernels") == "chain" and self.allow_chain and self.num_layers > 0
                and not self.ragged and not self.p.fp8 and not cfg.is_moe
                and B <= min(4, gemv_max_rows()) and cfg.n_kv_heads * B <= 60 and cfg.n_heads // cfg.n_kv_heads <= 8
                and cfg.head_dim in (64, 128) and self._chain_ring_fits(B))

    def _chain_ring_fits(self, B: int) -> bool:
        """The chain launcher places B rows of the widest input (the down projection's) beside its weight ring; at
        Qwen2.5-7B width four rows leave too little shared memory for the ring, and such steps take the per-kernel
        sequence."""
        cfg = self.cfg
        return nat.decode_chain_geometry(B, max(cfg.hidden, cfg.q_dim, cfg.intermediate)) is not None

    def _chain_group(self) -> int:
        """Decoder layers per chain launch (TL_CHAIN_LAYERS, default 1; 5 jobs per layer, at most 3 layers)."""
        import os
        return max(1, min(3, int(os.environ.get("TL_CHAIN_LAYERS", "1"))))

    def _decode_chains(self, x: torch.Tensor, B: int, out: Optional[torch.Tensor]):
        """The launch list of one decode step of this shard: qkv of the first layer as a stand-alone GEMV, then one
        persistent launch per group of layers [ATTN, o, gate/up, down, qkv of the next layer]."""
        key = (B, x.data_ptr(), 0 if out is None else out.data_ptr())
        if key in self._chains:
            return self._chains[key]
        cfg, v = self.cfg, self.p.v
        w = self._dbufs(B)
        J = nat.make_job
        if self.chain_sync is None:
            self.chain_sync = torch.zeros(self.num_layers + 1, nat.CHAIN_SYNC_BYTES // 4, dtype=torch.int32, device=self.device)
            self.chain_attn_ws = torch.empty(nat.decode_chain_ws(min(self.B_max, 4), cfg.n_heads, cfg.n_kv_heads, cfg.head_dim),
                                             dtype=torch.uint8, device=self.device)
        per = self._chain_group()
        launches = []
        for g0 in range(0, self.num_layers, per):
            jobs = []
            g1 = min(self.num_layers, g0 + per)
            for j in range(g0, g1):
                li = self.layer_ids[j]
                jobs.append(J(nat.JOB_ATTN, x=w.qkv, y=w.attn, k_cache=self.kc[j], v_cache=self.vc[j], pos_dev=self.pos_dev,
                              cos_tab=self.cos, sin_tab=self.sin, q_norm_w=v.get(f"l{li}.qn"), k_norm_w=v.get(f"l{li}.kn"),
                              n_h=cfg.n_heads, n_kv=cfg.n_kv_heads, d=cfg.head_dim, T_max=self.T_max, scale=self.scale,
                              eps=cfg.rms_eps))
                jobs.append(J(nat.JOB_GEMV, N=cfg.hidden, K=cfg.q_dim, flags=nat.EPI_RESIDUAL, W=v[f"l{li}.wo"], x=w.attn, y=x,
                              residual=x))
                jobs.append(J(nat.JOB_GEMV, N=2 * cfg.intermediate, K=cfg.hidden, flags=nat.EPI_SWIGLU, W=v[f"l{li}.wgu"], x=x,
                              y=w.act, norm_w=v[f"l{li}.ln2"], eps=cfg.rms_eps))
                last = j == self.num_layers - 1
                jobs.append(J(nat.JOB_GEMV, N=cfg.hidden, K=cfg.intermediate, flags=nat.EPI_RESIDUAL, W=v[f"l{li}.wd"], x=w.act,
                              y=(out if (last and out is not None) else x), residual=x))
                if not last:
                    ln = self.layer_ids[j + 1]
                    bq = v.get(f"l{ln}.bqkv")
                    jobs.append(J(nat.JOB_GEMV, N=cfg.qkv_dim, K=cfg.hidden, flags=nat.EPI_BIAS if bq is not None else 0,
                                  W=v[f"l{ln}.wqkv"], x=x, y=w.qkv, bias=bq, norm_w=v[f"l{ln}.ln1"], eps=cfg.rms_eps))
            # what the launch after this one streams first: the next group's o-projection, or whatever follows the shard
            nxt = v[f"l{self.layer_ids[g1]}.wo"] if g1 < self.num_layers else self.weights_after_last_layer
            launches.append(nat.DecodeChain(jobs, B, self.chain_sync[g0 // per], self.chain_attn_ws, nxt))
        self._chains[key] = launches
        return launches

    def _decode_step_chained(self, x: torch.Tensor, B: int, out: Optional[torch.Tensor]):
        cfg, v = self.cfg, self.p.v
        w = self._dbufs(B)
        l0 = self.layer_ids[0]
        nat.gemv(x, v[f"l{l0}.wqkv"], out=w.qkv, bias=v.get(f"l{l0}.bqkv"), norm_w=v[f"l{l0}.ln1"], eps=cfg.rms_eps,
                 next_w=v[f"l{l0}.wo"])
        for ch in self._decode_chains(x, B, out):
            ch.launch()

    def dq_ok(self, B: int) -> bool:
        """TL_DECODE_IMPL=dq: the per-kernel sequence, except that the down projection of layer j and the qkv projection
        of layer j+1 run as ONE two-job chain launch (one software dependency instead of a launch boundary between a
        long and a short weight stream)."""
        import os
        return (os.environ.get("TL_DECODE_IMPL", "kernels") == "dq" and self.allow_chain and self.num_layers > 1
                and B <= min(4, gemv_max_rows()) and not self.p.fp8 and not self.cfg.is_moe and self._chain_ring_fits(B))

    def _decode_step_dq(self, x: torch.Tensor, B: int, out: Optional[torch.Tensor]):
        cfg, v = self.cfg, self.p.v
        w = self._dbufs(B)
        key = ("dq", B, x.data_ptr(), 0 if out is None else out.data_ptr())
        if key not in self._chains:
            J = nat.make_job
            if self.chain_sync is None:
                self.chain_sync = torch.zeros(self.num_layers + 1, nat.CHAIN_SYNC_BYTES // 4, dtype=torch.int32, device=self.device)
                self.chain_attn_ws = torch.empty(nat.decode_chain_ws(min(self.B_max, 4), cfg.n_heads, cfg.n_kv_heads, cfg.head_dim),
                                                 dtype=torch.uint8, device=self.device)
            launches = []
            for j in range(self.num_layers - 1):
                li, ln = self.layer_ids[j], self.layer_ids[j + 1]
                bq = v.get(f"l{ln}.bqkv")
                jobs = [J(nat.JOB_GEMV, N=cfg.hidden, K=cfg.intermediate, flags=nat.EPI_RESIDUAL, W=v[f"l{li}.wd"], x=w.act, y=x, residual=x),
                        J(nat.JOB_GEMV, N=cfg.qkv_dim, K=cfg.hidden, flags=nat.EPI_BIAS if bq is not None else 0, W=v[f"l{ln}.wqkv"], x=x,
                          y=w.qkv, bias=bq, norm_w=v[f"l{ln}.ln1"], eps=cfg.rms_eps)]
                launches.append(nat.DecodeChain(jobs, B, self.chain_sync[j], self.chain_attn_ws, v[f"l{ln}.wo"]))
            self._chains[key] = launches
        chains = self._chains[key]
        l0 = self.layer_ids[0]
        nat.gemv(x, v[f"l{l0}.wqkv"], out=w.qkv, bias=v.get(f"l{l0}.bqkv"), norm_w=v[f"l{l0}.ln1"], eps=cfg.rms_eps, next_w=v[f"l{l0}.wo"])
        for j, li in enumerate(self.layer_ids):
            self._decode_attention(j, li, B, w)
            nat.gemv(w.attn, v[f"l{li}.wo"], out=x, residual=x, next_w=v[f"l{li}.wgu"])
            nat.gemv(x, v[f"l{li}.wgu"], out=w.act, norm_w=v[f"l{li}.ln2"], eps=cfg.rms_eps, flags=nat.EPI_SWIGLU, next_w=v[f"l{li}.wd"])
            if j + 1 < self.num_layers:
                chains[j].launch()
            else:
                nat.gemv(w.act, v[f"l{li}.wd"], out=x if out is None else out, residual=x, next_w=self.weights_after_last_layer)

    def n_chain_launches(self) -> int:
        per = self._chain_group()
        return 1 + (self.num_layers + per - 1) // per

    def check(self):
        """Raise if a chain launch gave up on a dependency wait (error word of its sync slot)."""
        if self.chain_sync is not None and int(self.chain_sync[:, 2].max().item()):
            self.chain_sync[:, :4].zero_()
            raise nat.NativeError("decode chain kernel timed out waiting for a dependency (co-residency of its CTAs lost?)")

    # ------------------------------------------------------------------------------------------ reference-shaped API
    def forward(self, **kwargs) -> dict:
        """``LayerGroupModule.forward`` contract (injector.py:252-260): returns kwargs ∪ outputs."""
        hs = kwargs["hidden_states"]
        past_len = int(kwargs.get("past_len", 0) or 0)
        out = dict(kwargs)
        out["hidden_states"] = self.prefill(hs, past_len).clone()
        return out

    __call__ = forward
