"""Training through the pipeline stages: forward with saved activations, hand-written backward, fused AdamW.

Reference semantics being replaced (/root/reference/tensorlink/ml):
  * ``DistributedModel.forward`` splits the batch into ``n_pipelines`` micro-batches (module.py:374-399) and wraps the
    output in ``CustomAutogradRouter`` so that ``loss.backward()`` reaches ``DistributedModel.backward`` (:126-144,
    :414-437), which walks the recorded shard boundaries LIFO and RPCs each gradient to its worker (:439-524);
  * the worker keeps ``{"inputs","output"}`` per micro-batch and runs ``assoc_output.backward(grad)`` over HF's
    autograd graph, returning the gradient of the shard input (worker.py:233-295, zeros where a grad is missing);
  * ``optimizer.step()`` / ``zero_grad()`` fan out to every worker (optim.py:131-187, worker.py:1309-1327).
Here each rank owns its stage's flat parameter and gradient arenas; the backward of a decoder layer is eight
wgmma GEMMs (dgrad + wgrad, MN-major operands, gradient accumulation in the epilogue) plus the attention /
norm / RoPE / SwiGLU backward kernels; gradients of ``hidden_states`` hop rank i+1 -> i over NVLink.  The loss and
its gradient are produced on the last stage by a fused lm_head + cross-entropy pass over token chunks, so the
[tokens, vocab] logits never exist in full (one micro-batch); in a pipelined step only logits + loss run in the forward
phase and the head's dgrad / wgrad join the backward chain / the deferred weight gradients (``head_loss_and_grad``).
The object returned as ``.loss`` is an autograd proxy on EVERY rank:
``loss.backward()`` runs that rank's part of the pipeline backward (SPMD equivalent of the autograd router).

Tied embeddings split over two ranks (Qwen2.5-0.5B at N > 1): the two copies' gradients are summed rank 0 <-> last
rank before the optimizer step, so both copies take identical updates.
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

from .. import native as nat
from .module import CausalLMOutput

A_MN, B_MN, ACC = nat.A_MN_MAJOR, nat.B_MN_MAJOR, nat.EPI_ACCUM
HEAD_CHUNK = 2048          # tokens per fused lm_head + CE pass
HEAD_STASH_BYTES = 32 << 30  # most d(logits) a pipelined step may keep for the split head backward (7B, 64 x 512: 10 GB)


class StageTrainer:
    """Training-mode execution of one ``CudaStage`` (activations saved per micro-batch).

    Weight gradients.  With one micro-batch a layer's four weight-gradient GEMMs follow its dgrad GEMMs directly.
    With several micro-batches in a step (``begin_step(n_mb > 1)``) the backward of a micro-batch runs the dgrad chain
    only and leaves (grad_out, input) of every Linear in per-layer stash buffers laid out [all tokens of the step, dim];
    ``weight_grads()`` then produces every weight gradient with ONE GEMM whose contraction runs over all tokens of the
    step.  That removes the per-micro-batch read-modify-write of the bf16 gradient arena (memory-bound for small
    micro-batches: 4 bytes per parameter against 2*tokens flops) and takes the weight gradients off the critical path
    of the pipeline: a stage that has finished its dgrads fills the drain of the pipeline with its weight gradients
    (the "deferred W" of zero-bubble schedules) while earlier stages are still receiving gradients.
    As soon as a layer's gradients are final an event is recorded, so the optimizer can update that layer on a side
    stream while the remaining weight-gradient GEMMs still run (``StageAdam.step``).

    Left-padded micro-batches (``kv_start``, see ``train_forward``) run the ``_rows`` attention forward and backward:
    keys below a row's start are never attended and pad tokens receive exact zeros from the attention backward."""

    supports_kv_start = True

    def __init__(self, stage):
        self.st = stage
        self.cfg = stage.cfg
        self.p = stage.params
        self.layer_ids = stage.params.layer_ids
        dev = stage.device
        names = [f"l{li}.{n}" for li in self.layer_ids for n in ("ln1", "ln2")] + (["norm"] if stage.has_head else [])
        self.norm_acc: Dict[str, torch.Tensor] = {n: torch.zeros(self.cfg.hidden, dtype=torch.float32, device=dev)
                                                  for n in names}
        if self.cfg.qkv_bias:
            for li in self.layer_ids:
                self.norm_acc[f"l{li}.bqkv"] = torch.zeros(self.cfg.qkv_dim, dtype=torch.float32, device=dev)
        if self.cfg.qk_norm:
            for li in self.layer_ids:
                for n in ("qn", "kn"):
                    self.norm_acc[f"l{li}.{n}"] = torch.zeros(self.cfg.head_dim, dtype=torch.float32, device=dev)
        self.grp = stage.slots[0]                     # rope tables / scale come from the shard operator
        self.ctx: Dict[int, dict] = {}
        self.loss_sum = torch.zeros(1, dtype=torch.float32, device=dev)
        self.n_valid_dev = torch.zeros(1, dtype=torch.int32, device=dev)
        self.launches = 0
        # Weight matrices whose gradient is produced by weight-gradient GEMMs only.  zero_grad() does not memset
        # them (99.9 % of the gradient arena): it marks them "fresh" and the first weight-gradient GEMM afterwards WRITES
        # the tensor instead of read-modify-writing zeros (saves the 15 GB memset and a 15 GB read per step at 7B).
        self._lazy = [f"l{li}.{n}" for li in self.layer_ids for n in ("wqkv", "wo", "wgu", "wd")]
        if stage.has_head and not (self.cfg.tied and stage.has_embed) and "head" in self.p.g and not self.cfg.tied:
            self._lazy.append("head")
        self._fresh: set = set()
        self._eager = [t for n, t in self.p.g.items() if n not in set(self._lazy)]
        self.p.grad_settle = self.settle_grads          # gradient export (hf_state_dict(grads=True)) settles first
        # ---- step state
        self.n_mb, self.tok_mb, self.defer_w = 1, 0, False
        self.stash: Dict[int, Dict[str, torch.Tensor]] = {}
        self._stash_key = None
        self.layer_events: Dict[int, torch.cuda.Event] = {}        # layer index j -> "gradients of layer j are final"
        self.final_order: List[int] = []
        self.params_ready: Optional[torch.cuda.Event] = None       # an optimizer update still running on a side stream
        self.overlap_ok = False                                    # layer_events describe a complete, regular step
        # lm_head / final-norm gradients are produced during the forward pass (fused with the loss) into PENDING
        # buffers and enter the gradient arena in backward(), multiplied by the upstream gradient: a forward that is
        # never followed by backward leaves the arena untouched, (loss * c).backward() scales them like everything else
        self.head_pending: Optional[torch.Tensor] = None
        self.head_norm_pending: Optional[torch.Tensor] = None
        self._head_pending_live = False
        self.head_split, self._head_w_done, self._head_scale = False, False, 1.0
        self.head_stash: Dict[str, torch.Tensor] = {}
        self.embed_pending: Optional[torch.Tensor] = None          # tied embedding on another rank than the head

    # ------------------------------------------------------------------------------------------ step set-up
    def wait_params(self):
        """Order the current stream after a side-stream optimizer update (parameters and gradients are shared)."""
        if self.params_ready is not None:
            torch.cuda.current_stream().wait_event(self.params_ready)
            self.params_ready = None

    def begin_step(self, n_mb: int, b: int, S: int):
        """Called by ``train_forward`` once per step on every rank: micro-batch geometry of this step."""
        self.wait_params()
        self.n_mb, self.tok_mb = n_mb, b * S
        self.defer_w = n_mb > 1
        self.layer_events, self.final_order = {}, []
        self._head_pending_live = False
        self.head_split = False
        if not self.defer_w:
            return
        key = (n_mb, self.tok_mb)
        if self._stash_key == key:
            self.head_split = bool(self.head_stash)
            return
        cfg, dev, bf = self.cfg, self.p.device, torch.bfloat16
        n = n_mb * self.tok_mb
        self.stash, self.head_stash = {}, {}
        torch.cuda.empty_cache()
        # the head's own backward leaves the forward phase when its d(logits) fit (see head_loss_and_grad); else the
        # fused, chunked form runs in the forward phase as in a single-micro-batch step
        need = n * cfg.vocab * 2
        self.head_split = (bool(self.st.has_head) and need <= HEAD_STASH_BYTES
                           and need <= torch.cuda.mem_get_info(dev)[0] // 2)
        if self.head_split:
            self.head_stash = {"hn": torch.empty(n, cfg.hidden, dtype=bf, device=dev),
                               "dlogits": torch.empty(n, cfg.vocab, dtype=bf, device=dev),
                               "rstd": torch.empty(n, dtype=torch.float32, device=dev)}
        for j in range(len(self.layer_ids)):
            self.stash[j] = {
                "h1": torch.empty(n, cfg.hidden, dtype=bf, device=dev), "attn": torch.empty(n, cfg.q_dim, dtype=bf, device=dev),
                "h2": torch.empty(n, cfg.hidden, dtype=bf, device=dev), "act": torch.empty(n, cfg.intermediate, dtype=bf, device=dev),
                "dy": torch.empty(n, cfg.hidden, dtype=bf, device=dev), "dgu": torch.empty(n, 2 * cfg.intermediate, dtype=bf, device=dev),
                "d_xmid": torch.empty(n, cfg.hidden, dtype=bf, device=dev), "dqkv": torch.empty(n, cfg.qkv_dim, dtype=bf, device=dev)}
        self._stash_key = key

    def _rows(self, mb) -> Optional[slice]:
        """Rows of the stash that belong to micro-batch ``mb`` (None: this call is not part of a deferred step)."""
        if self.defer_w and isinstance(mb, int) and 0 <= mb < self.n_mb:
            return slice(mb * self.tok_mb, (mb + 1) * self.tok_mb)
        return None

    def grad_in_buffer(self, mb, b: int, S: int) -> torch.Tensor:
        """Where the gradient of this stage's output for micro-batch ``mb`` should land (receive buffer): the stash
        rows of the last layer when weight gradients are deferred, so the hop needs no extra copy."""
        r = self._rows(mb)
        if r is not None and b * S == self.tok_mb and len(self.layer_ids):
            return self.stash[len(self.layer_ids) - 1]["dy"][r].view(b, S, self.cfg.hidden)
        return torch.empty(b, S, self.cfg.hidden, dtype=torch.bfloat16, device=self.p.device)

    # ------------------------------------------------------------------------------------------ forward
    def forward_layers(self, mb, x: torch.Tensor, kv_start: Optional[torch.Tensor] = None) -> torch.Tensor:
        """x [b,S,H] -> [b,S,H] through this stage's layers, saving what the backward needs.  ``kv_start`` (int32[b] on
        the device, optional): leading pad tokens of each row, whose keys no query attends to (RoPE positions stay
        0..S-1 in every row, as in HF's training forward)."""
        cfg, v = self.cfg, self.p.v
        b, S, H = x.shape
        N = b * S
        dev, bf = x.device, torch.bfloat16
        x = x.reshape(N, H).contiguous()
        saved: List[dict] = []
        rows = self._rows(mb) if N == self.tok_mb else None
        zero_pos = torch.zeros(1, dtype=torch.int32, device=dev)
        for j, li in enumerate(self.layer_ids):
            st = self.stash[j] if rows is not None else None
            s = {"x_in": x}
            s["rstd1"] = torch.empty(N, dtype=torch.float32, device=dev)
            s["h1"] = nat.rmsnorm_fwd(x, v[f"l{li}.ln1"], cfg.rms_eps, rstd=s["rstd1"], out=st["h1"][rows] if st else None)
            qkv = nat.gemm(s["h1"], v[f"l{li}.wqkv"], bias=v.get(f"l{li}.bqkv"))
            s["q"] = torch.empty(N, cfg.q_dim, dtype=bf, device=dev)
            s["kc"] = torch.empty(b, cfg.n_kv_heads, S, cfg.head_dim, dtype=bf, device=dev)
            s["vc"] = torch.empty_like(s["kc"])
            if cfg.qk_norm:
                s["qkv"] = qkv                      # pre-norm q/k are needed by the q/k-norm backward
            nat.rope_kv_fwd(qkv, s["q"], s["kc"], s["vc"], zero_pos, self.grp.cos, self.grp.sin, v.get(f"l{li}.qn"),
                            v.get(f"l{li}.kn"), cfg.rms_eps, S, cfg.n_heads, cfg.n_kv_heads, cfg.head_dim)
            s["attn"] = st["attn"][rows] if st else torch.empty(N, cfg.q_dim, dtype=bf, device=dev)
            s["lse"] = torch.empty(b, cfg.n_heads, S, dtype=torch.float32, device=dev)
            nat.attn_prefill_fwd(s["q"], s["kc"], s["vc"], s["attn"], s["lse"], b, S, 0, cfg.n_heads, cfg.n_kv_heads,
                                 cfg.head_dim, self.grp.scale, kv_start=kv_start)
            s["x_mid"] = nat.gemm(s["attn"], v[f"l{li}.wo"], residual=x)
            s["rstd2"] = torch.empty(N, dtype=torch.float32, device=dev)
            s["h2"] = nat.rmsnorm_fwd(s["x_mid"], v[f"l{li}.ln2"], cfg.rms_eps, rstd=s["rstd2"], out=st["h2"][rows] if st else None)
            s["gu"] = nat.gemm(s["h2"], v[f"l{li}.wgu"])
            s["act"] = st["act"][rows] if st else torch.empty(N, cfg.intermediate, dtype=bf, device=dev)   # the down-proj wgrad needs it
            nat.swiglu_fwd(s["gu"], s["act"])
            x = nat.gemm(s["act"], v[f"l{li}.wd"], residual=s["x_mid"])
            saved.append(s)
            self.launches += 10
        self.ctx[mb] = {"layers": saved, "b": b, "S": S, "deferred": rows is not None, "kv_start": kv_start}
        return x.view(b, S, H)

    def head_loss_and_grad(self, mb, x: torch.Tensor, shift_labels: torch.Tensor, inv_n: float) -> None:
        """Last stage: final norm + lm_head + shifted CE, fused with its own backward, chunked over tokens.
        Accumulates the loss sum, stores d(loss)/d(x) for ``backward`` and leaves the lm_head / final-norm gradients of
        this forward in the PENDING buffers (``commit_head`` adds them to the arena with the upstream scale)."""
        cfg, v = self.cfg, self.p.v
        b, S, H = x.shape
        N = b * S
        x2 = x.reshape(N, H)
        labels = shift_labels.reshape(N).contiguous()
        if self.head_pending is None:
            self.head_pending = torch.empty(cfg.vocab, H, dtype=torch.bfloat16, device=x.device)
            self.head_norm_pending = torch.zeros(H, dtype=torch.float32, device=x.device)
        rows = self._rows(mb) if (self.head_split and N == self.tok_mb) else None
        if rows is not None:
            # Pipelined step: only logits + loss here.  The fused form below puts 3 lm_head-sized GEMMs (7 decoder layers'
            # worth of forward work at 7B) into the last stage's FORWARD phase, which every other stage then waits for
            # before the first gradient can flow back; split, the forward phase carries one of them, the dgrad chain one
            # (``head_backward``) and the weight gradient joins the deferred ones (``weight_grads``), one GEMM over all
            # tokens.  d(logits) replace the logits in place and stay in the stash until then.
            hs = self.head_stash
            nat.rmsnorm_fwd(x2, v["norm"], cfg.rms_eps, rstd=hs["rstd"][rows], out=hs["hn"][rows])
            logits = nat.gemm(hs["hn"][rows], v["head"], out=hs["dlogits"][rows])
            nat.ce_fwd_bwd(logits, labels, self.loss_sum, self.n_valid_dev, logits, inv_n)
            if not self._head_pending_live:
                self.head_norm_pending.zero_()
                self._head_pending_live = True
            self.ctx[mb]["x_out"] = x2
            self.launches += 3
            return
        dx = torch.empty_like(x2)
        for a in range(0, N, HEAD_CHUNK):
            e = min(N, a + HEAD_CHUNK)
            xc = x2[a:e]
            rstd = torch.empty(e - a, dtype=torch.float32, device=x.device)
            hn = nat.rmsnorm_fwd(xc, v["norm"], cfg.rms_eps, rstd=rstd)
            logits = nat.gemm(hn, v["head"])
            nat.ce_fwd_bwd(logits, labels[a:e], self.loss_sum, self.n_valid_dev, logits, inv_n)
            dhn = nat.gemm(logits, v["head"], flags=B_MN, N=H)                       # [n,V]·[V,H]
            first = not self._head_pending_live
            if first:
                self.head_norm_pending.zero_()
                self._head_pending_live = True
            nat.gemm(logits, hn, out=self.head_pending, flags=A_MN | B_MN | (0 if first else ACC), M=cfg.vocab, K=e - a, N=H)   # dW (+)= dlogits^T·hn
            nat.rmsnorm_bwd(xc, v["norm"], dhn, rstd, dx[a:e], self.head_norm_pending)
            self.launches += 6
        self.ctx[mb]["dx_out"] = dx.view(b, S, H)

    def head_backward(self, mb, scale: float) -> torch.Tensor:
        """Last stage, start of the dgrad chain of micro-batch ``mb``: gradient of the stage's last hidden state — from the
        fused forward (``dx_out``), or, in a split step, d(logits)·W_head and the final norm's backward now."""
        c = self.ctx[mb]
        if "dx_out" in c:
            dy = c.pop("dx_out")
            return dy * scale if scale != 1.0 else dy
        cfg, v, hs, rows = self.cfg, self.p.v, self.head_stash, self._rows(mb)
        x2 = c.pop("x_out")
        dhn = nat.gemm(hs["dlogits"][rows], v["head"], flags=B_MN, N=cfg.hidden)          # [n,V]·[V,H]
        dx = torch.empty_like(x2)
        nat.rmsnorm_bwd(x2, v["norm"], dhn, hs["rstd"][rows], dx, self.head_norm_pending)
        self.launches += 2
        if scale != 1.0:
            dx = dx * scale
        return dx.view(c["b"], c["S"], cfg.hidden)

    def commit_head(self, scale: float) -> Optional[torch.Tensor]:
        """backward() on the last stage: pending lm_head / final-norm gradients x upstream gradient -> arena.
        Returns the scaled lm_head gradient of THIS backward (the tied-embedding exchange needs the delta alone).
        In a split step this runs after the dgrad chains (from ``weight_grads``), once the pending buffers are complete."""
        if not self._head_pending_live:
            return None
        if self.head_split and not self._head_w_done:
            self._head_scale = scale             # nothing to commit yet: weight_grads() produces the gradient, then commits
            return None
        self._head_pending_live = False
        if self.cfg.tied and not self.st.has_embed:
            # the tied copy lives on rank 0: the caller exchanges deltas, nothing enters the arena here
            if scale != 1.0:
                nat.scale_add(self.head_pending.view(-1), self.head_pending.view(-1), scale, accumulate=False)
        else:
            nat.scale_add(self.p.g["head"].view(-1), self.head_pending.view(-1), scale, accumulate=not self._take_fresh("head"))
        nat.scale_add(self.norm_acc["norm"], self.head_norm_pending, scale, accumulate=True)
        self.launches += 2
        return self.head_pending

    # ------------------------------------------------------------------------------------------ backward
    def backward_layers(self, mb, dy: torch.Tensor) -> torch.Tensor:
        """dy [b,S,H] (gradient of this stage's output) -> gradient of its input.  Parameter gradients accumulate here
        (one micro-batch per step, or calls outside a step: the worker surface) or in ``weight_grads`` (deferred)."""
        cfg, v, g = self.cfg, self.p.v, self.p.g
        c = self.ctx.pop(mb)
        self.overlap_ok = False                      # (train_backward sets it again once the whole step is through)
        b, S = c["b"], c["S"]
        N, H = b * S, cfg.hidden
        dev, bf = dy.device, torch.bfloat16
        rows = self._rows(mb) if c.get("deferred") else None
        dy = dy.reshape(N, H)
        if not dy.is_contiguous():
            dy = dy.contiguous()
        ws = torch.empty(max(nat.attn_bwd_ws(b, S, cfg.n_heads), 16), dtype=torch.uint8, device=dev)
        n_layers = len(self.layer_ids)
        for j in reversed(range(n_layers)):
            li, s = self.layer_ids[j], c["layers"][j]
            st = self.stash[j] if rows is not None else None
            if st is not None and dy.data_ptr() != st["dy"][rows].data_ptr():
                st["dy"][rows].copy_(dy)                 # (the last layer's dy normally arrives in place: grad_in_buffer)
                dy = st["dy"][rows]
            # ---- MLP
            act = s["act"]
            d_act = nat.gemm(dy, v[f"l{li}.wd"], flags=B_MN, N=cfg.intermediate)         # dy·Wd
            if st is None:
                nat.gemm(dy, act, out=g[f"l{li}.wd"], flags=A_MN | B_MN | self._acc(f"l{li}.wd"), M=H, K=N, N=cfg.intermediate)
            dgu = st["dgu"][rows] if st else torch.empty_like(s["gu"])
            nat.swiglu_bwd(s["gu"], d_act, dgu)
            dh2 = nat.gemm(dgu, v[f"l{li}.wgu"], flags=B_MN, N=H)
            if st is None:
                nat.gemm(dgu, s["h2"], out=g[f"l{li}.wgu"], flags=A_MN | B_MN | self._acc(f"l{li}.wgu"), M=2 * cfg.intermediate, K=N, N=H)
            d_xmid = st["d_xmid"][rows] if st else torch.empty(N, H, dtype=bf, device=dev)
            nat.rmsnorm_bwd(s["x_mid"], v[f"l{li}.ln2"], dh2, s["rstd2"], d_xmid, self.norm_acc[f"l{li}.ln2"], dx_add=dy)
            # ---- attention
            d_attn = nat.gemm(d_xmid, v[f"l{li}.wo"], flags=B_MN, N=cfg.q_dim)
            if st is None:
                nat.gemm(d_xmid, s["attn"], out=g[f"l{li}.wo"], flags=A_MN | B_MN | self._acc(f"l{li}.wo"), M=H, K=N, N=cfg.q_dim)
            dq = torch.empty(N, cfg.q_dim, dtype=bf, device=dev)
            dk = torch.empty(b, cfg.n_heads, S, cfg.head_dim, dtype=bf, device=dev)     # one partial per query head
            dv = torch.empty_like(dk)
            nat.attn_bwd(s["q"], s["kc"], s["vc"], s["attn"], d_attn, s["lse"], dq, dk, dv, ws, b, S, cfg.n_heads,
                         cfg.n_kv_heads, cfg.head_dim, self.grp.scale, kv_start=c.get("kv_start"))
            dqkv = st["dqkv"][rows] if st else torch.empty(N, cfg.qkv_dim, dtype=bf, device=dev)
            nat.rope_kv_bwd(dq, dk, dv, dqkv, self.grp.cos, self.grp.sin, S, cfg.n_heads, cfg.n_kv_heads, cfg.head_dim)
            if cfg.qk_norm:
                nat.qk_norm_bwd(s["qkv"], dqkv, v[f"l{li}.qn"], v[f"l{li}.kn"], self.norm_acc[f"l{li}.qn"],
                                self.norm_acc[f"l{li}.kn"], cfg.rms_eps, cfg.n_heads, cfg.n_kv_heads, cfg.head_dim)
            dh1 = nat.gemm(dqkv, v[f"l{li}.wqkv"], flags=B_MN, N=H)
            if st is None:
                nat.gemm(dqkv, s["h1"], out=g[f"l{li}.wqkv"], flags=A_MN | B_MN | self._acc(f"l{li}.wqkv"), M=cfg.qkv_dim, K=N, N=H)
                if cfg.qkv_bias:
                    nat.colsum(dqkv, self.norm_acc[f"l{li}.bqkv"])
            # the layer below reads this as its dy: write it where its weight-gradient GEMM will look for it
            dx = (self.stash[j - 1]["dy"][rows] if (st is not None and j > 0) else torch.empty(N, H, dtype=bf, device=dev))
            nat.rmsnorm_bwd(s["x_in"], v[f"l{li}.ln1"], dh1, s["rstd1"], dx, self.norm_acc[f"l{li}.ln1"], dx_add=d_xmid)
            dy = dx
            self.launches += 17 if st is None else 12
            if st is None and self.n_mb == 1 and isinstance(mb, int):
                self._finalize_layer(j)          # single micro-batch step: this layer's gradients are final now
        return dy.view(b, S, H)

    def weight_grads(self):
        """Deferred mode: every weight gradient of the stage as ONE GEMM over all tokens of the step (layers in the
        order their dgrads finished, so the optimizer can start on the first ones while the rest still run)."""
        if not self.defer_w:
            return
        cfg, g = self.cfg, self.p.g
        H, n = cfg.hidden, self.n_mb * self.tok_mb
        if self.head_split and self._head_pending_live:
            hs = self.head_stash
            nat.gemm(hs["dlogits"], hs["hn"], out=self.head_pending, flags=A_MN | B_MN, M=cfg.vocab, K=n, N=H)   # dW = dlogits^T·hn
            self.launches += 1
            self._head_w_done = True
            self.commit_head(self._head_scale)
            self._head_w_done = False
        for j in reversed(range(len(self.layer_ids))):
            li, st = self.layer_ids[j], self.stash[j]
            nat.gemm(st["dy"], st["act"], out=g[f"l{li}.wd"], flags=A_MN | B_MN | self._acc(f"l{li}.wd"), M=H, K=n, N=cfg.intermediate)
            nat.gemm(st["dgu"], st["h2"], out=g[f"l{li}.wgu"], flags=A_MN | B_MN | self._acc(f"l{li}.wgu"), M=2 * cfg.intermediate, K=n, N=H)
            nat.gemm(st["d_xmid"], st["attn"], out=g[f"l{li}.wo"], flags=A_MN | B_MN | self._acc(f"l{li}.wo"), M=H, K=n, N=cfg.q_dim)
            nat.gemm(st["dqkv"], st["h1"], out=g[f"l{li}.wqkv"], flags=A_MN | B_MN | self._acc(f"l{li}.wqkv"), M=cfg.qkv_dim, K=n, N=H)
            if cfg.qkv_bias:
                nat.colsum(st["dqkv"], self.norm_acc[f"l{li}.bqkv"])
            self.launches += 5 if cfg.qkv_bias else 4
            self._finalize_layer(j)

    def _layer_small_names(self, li: int) -> List[str]:
        return [n for n in (f"l{li}.ln1", f"l{li}.ln2", f"l{li}.bqkv", f"l{li}.qn", f"l{li}.kn") if n in self.norm_acc]

    def _finalize_layer(self, j: int):
        """Fold the fp32 accumulators of layer j (norm gains, bias, q/k-norm gains) into the bf16 arena and mark the
        layer's gradients final."""
        for n in self._layer_small_names(self.layer_ids[j]):
            nat.f32_to_bf16_accum(self.norm_acc[n], self.p.g[n], accumulate=True)
            self.norm_acc[n].zero_()
        ev = torch.cuda.Event()
        ev.record()
        self.layer_events[j] = ev
        self.final_order.append(j)

    def embed_backward(self, ids: torch.Tensor, dx: torch.Tensor, into: Optional[torch.Tensor] = None):
        nat.embed_bwd(ids.reshape(-1).contiguous(), dx.reshape(-1, self.cfg.hidden).contiguous(),
                      self.p.g["embed"] if into is None else into)
        self.launches += 1

    def finish_backward(self):
        """fold what is left of the fp32 accumulators into the bf16 gradient arena"""
        self.settle_grads()
        done = {n for j in self.layer_events for n in self._layer_small_names(self.layer_ids[j])}
        for n, acc in self.norm_acc.items():
            if n in done:
                continue
            nat.f32_to_bf16_accum(acc, self.p.g[n], accumulate=True)
            acc.zero_()

    def _take_fresh(self, name: str) -> bool:
        if name in self._fresh:
            self._fresh.discard(name)
            return True
        return False

    def _acc(self, name: str) -> int:
        """EPI_ACCUM unless this is the first gradient GEMM into ``name`` since zero_grad()."""
        return 0 if self._take_fresh(name) else ACC

    def settle_grads(self):
        """Give every still-fresh (never written since zero_grad) matrix gradient its zeros: called before anything reads
        the gradient arena as a whole (optimizer step, gradient export)."""
        for n in self._fresh:
            self.p.g[n].zero_()
        self._fresh.clear()

    def zero_grad(self):
        self.wait_params()
        torch._foreach_zero_(self._eager)
        self._fresh = set(self._lazy)
        for a in self.norm_acc.values():
            a.zero_()


class _PipelineRouter(torch.autograd.Function):
    """SPMD counterpart of the reference's ``CustomAutogradRouter`` (module.py:126-144)."""

    @staticmethod
    def forward(ctx, anchor, dm, value):
        ctx.dm = dm
        return value.clone()

    @staticmethod
    def backward(ctx, grad_out):
        train_backward(ctx.dm, float(grad_out))
        return torch.zeros(()), None, None


def _trainer(dm) -> StageTrainer:
    if getattr(dm.stage, "trainer", None) is None:
        make = getattr(dm.stage, "make_trainer", None)          # test backends provide their own twin
        dm.stage.trainer = make() if make else StageTrainer(dm.stage)
    return dm.stage.trainer


def train_forward(dm, input_ids: Optional[torch.Tensor], labels: Optional[torch.Tensor],
                  padding: Optional[Tuple[List[int], torch.Tensor]] = None) -> CausalLMOutput:
    """Forward of all micro-batches (GPipe order).  Every rank returns an autograd proxy as ``.loss``.

    ``padding`` (first rank; ``module._train_mask`` of the ``attention_mask``): (kv_start, real) of a padded batch.
    A real query attends to the real keys of its row at or before it; RoPE positions stay 0..S-1 in every row, as in
    HF's forward without ``position_ids``.  Left padding masks keys below ``kv_start[b]`` in the attention kernels;
    right padding needs no kernel change (the causal mask already hides those keys from real queries).
    Deviation from HF: every label predicted FROM a pad position is ignored (the shifted label at t becomes -100
    where ``attention_mask[b, t] == 0``).  For right padding that is what collators already write; for left padding it
    drops one term per row, the first real token predicted from the last pad, whose HF logits come from a fully
    masked query row and differ between HF's attention backends.  Pad positions then carry no loss and real positions
    never read them, so pad tokens get exactly zero gradient."""
    link, st, cfg, dev = dm.link, dm.stage, dm.cfg, dm.device
    tr = _trainer(dm)
    meta = None
    if link.first:
        if labels is None:
            raise ValueError("training forward needs labels= (the loss is produced on the last stage)")
        B, S = input_ids.shape
        shift = F.pad(labels, (0, 1), value=-100)[:, 1:].contiguous()
        starts = None
        if padding is not None:
            starts, real = padding
            shift = shift.masked_fill(~real.to(shift.device), -100)
            if not any(starts):
                starts = None                    # right padding only: the plain kernels, exactly as an unpadded batch
        meta = (B, S, int((shift != -100).sum()), starts)
    B, S, n_valid, starts = link.broadcast_object(meta)
    if starts is not None and not getattr(tr, "supports_kv_start", False):
        raise NotImplementedError("left-padded training batches need a stage trainer with per-row key starts")
    n_mb = min(dm.n_pipelines, B)
    if B % n_mb:
        raise ValueError(f"batch {B} not divisible into {n_mb} micro-batches")
    b = B // n_mb
    if hasattr(tr, "begin_step"):
        tr.begin_step(n_mb, b, S)
    if link.first:
        ids_dev, shift_dev = input_ids.to(dev), shift.to(dev)
        if dm.world > 1:
            link.send_down(shift_dev, dm.world - 1)
    elif link.last:
        shift_dev = torch.empty(B, S, dtype=torch.int64, device=dev)
        link.recv_down(shift_dev, 0)
    tr.loss_sum.zero_()
    tr.n_valid_dev.zero_()
    dm._train_state = {"n_mb": n_mb, "b": b, "S": S, "ids": ids_dev if link.first else None}
    for m in range(n_mb):
        if link.first:
            x = st.embed(ids_dev[m * b:(m + 1) * b])
        else:
            x = torch.empty(b, S, cfg.hidden, dtype=torch.bfloat16, device=dev)
            link.recv_prev(x)
        mb_starts = starts[m * b:(m + 1) * b] if starts is not None else None
        if mb_starts is not None and any(mb_starts):
            x = tr.forward_layers(m, x, kv_start=torch.tensor(mb_starts, dtype=torch.int32, device=dev))
        else:
            x = tr.forward_layers(m, x)
        if not link.last:
            link.send_next(x.contiguous())
        else:
            tr.head_loss_and_grad(m, x, shift_dev[m * b:(m + 1) * b], 1.0 / max(n_valid, 1))
    loss = torch.zeros(1, dtype=torch.float32, device=dev)
    if link.last:
        loss = tr.loss_sum / max(n_valid, 1)
    if dm.world > 1:
        link.broadcast(loss, dm.world - 1)
    anchor = torch.zeros((), requires_grad=True)
    proxy = _PipelineRouter.apply(anchor, dm, loss.detach().float().cpu().reshape(()))
    return CausalLMOutput(loss=proxy, logits=None)


def train_backward(dm, grad_scale: float = 1.0):
    """Pipeline backward, micro-batches in reverse (module.py:414-524 / worker.py:233-295): the dgrad chain of every
    micro-batch first (the only part other stages wait for), then this stage's weight gradients."""
    link, st, cfg, dev = dm.link, dm.stage, dm.cfg, dm.device
    tr = _trainer(dm)
    s = dm._train_state
    tied_split = cfg.tied and dm.world > 1 and (link.first or link.last)
    head_delta = None
    if link.last and hasattr(tr, "commit_head"):
        head_delta = tr.commit_head(grad_scale)
    embed_into = None
    if tied_split and link.first and hasattr(tr, "embed_pending"):
        # this backward's embedding gradient alone (the exchange below must not re-send earlier accumulations)
        if tr.embed_pending is None:
            tr.embed_pending = torch.empty_like(st.params.g["embed"])
        tr.embed_pending.zero_()
        embed_into = tr.embed_pending
    for m in reversed(range(s["n_mb"])):
        if link.last and hasattr(tr, "head_backward"):
            dy = tr.head_backward(m, grad_scale)
        elif link.last:
            dy = tr.ctx[m].pop("dx_out")
            if grad_scale != 1.0:
                dy = dy * grad_scale
        else:
            dy = (tr.grad_in_buffer(m, s["b"], s["S"]) if hasattr(tr, "grad_in_buffer") else
                  torch.empty(s["b"], s["S"], cfg.hidden, dtype=torch.bfloat16, device=dev))
            link.recv_next(dy)
        dx = tr.backward_layers(m, dy)
        if not link.first:
            link.send_prev(dx.contiguous())
        elif embed_into is not None:
            tr.embed_backward(s["ids"][m * s["b"]:(m + 1) * s["b"]], dx, into=embed_into)
        else:
            tr.embed_backward(s["ids"][m * s["b"]:(m + 1) * s["b"]], dx)
    link.flush()
    if hasattr(tr, "weight_grads"):
        tr.weight_grads()
        if link.last and head_delta is None and getattr(tr, "head_split", False):
            head_delta = tr.head_pending         # split step: the lm_head gradient of this backward exists only now
    tr.finish_backward()
    if tied_split:
        # module.py:1218-1265 ties lm_head to embed_tokens on the host; here the two copies live on different ranks.
        # Both ranks add the SAME delta (this backward's embedding gradient + this backward's lm_head gradient) to
        # their copy, so repeated backward() calls without zero_grad() accumulate correctly and the copies stay equal.
        p = st.params
        if hasattr(tr, "embed_pending"):
            if link.last:
                link.send_up(head_delta, 0)
                eg = torch.empty_like(head_delta)
                link.recv_down(eg, 0)
                link.flush()
                nat.add_inplace(head_delta.view(-1), eg.view(-1))                      # delta = head part + embed part
                nat.add_inplace(p.g["head"].view(-1), head_delta.view(-1))
            else:
                hg = torch.empty_like(tr.embed_pending)
                link.recv_up(hg, dm.world - 1)
                link.send_down(tr.embed_pending.clone(), dm.world - 1)
                link.flush()
                nat.add_inplace(hg.view(-1), tr.embed_pending.view(-1))                # same sum (addition commutes)
                nat.add_inplace(p.g["embed"].view(-1), hg.view(-1))
        else:                                      # test twin without pending buffers: plain sum of the two arenas
            if link.last:
                link.send_up(p.g["head"], 0)
                link.flush()
                link.recv_down(p.g["head"], 0)
            else:
                tmp = torch.empty_like(p.g["embed"])
                link.recv_up(tmp, dm.world - 1)
                p.g["embed"].add_(tmp)
                link.send_down(p.g["embed"], dm.world - 1)
                link.flush()
    if hasattr(tr, "layer_events"):
        tr.overlap_ok = len(tr.layer_events) == len(tr.layer_ids)


class StageAdam:
    """``create_optimizer(**kw)`` result: ``step()`` / ``zero_grad()`` over this rank's arena (optim.py:131-187).

    ``step()`` after a regular ``loss.backward()`` updates layer by layer on a side stream: layer j's update waits only
    for the event "gradients of layer j are final" (recorded between the weight-gradient GEMMs), so the HBM-bound Adam
    sweep (22 bytes per parameter) runs under the remaining tensor-core-bound weight-gradient GEMMs instead of after
    them; the calling stream is ordered after the update before ``step()`` returns."""

    def __init__(self, dm, decoupled: bool = False, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0, **_):
        self.dm, self.decoupled = dm, decoupled
        self.lr, self.betas, self.eps, self.wd = lr, betas, eps, weight_decay
        p = dm.stage.params
        if p.grad is None:
            raise RuntimeError("DistributedModel was built with training=False; no gradient arena")
        self.m = torch.zeros(p.numel, dtype=torch.float32, device=p.device)
        self.v = torch.zeros_like(self.m)
        self.t = 0
        self.side: Optional[torch.cuda.Stream] = None
        self.param_groups = [{"lr": lr, "betas": betas, "eps": eps, "weight_decay": weight_decay}]   # scheduler surface

    def zero_grad(self, set_to_none: bool = False):
        _trainer(self.dm).zero_grad()

    def _update(self, a: int, e: int):
        p = self.dm.stage.params
        lr = self.param_groups[0]["lr"]
        nat.adamw_step(p.flat[a:e], p.grad[a:e], self.m[a:e], self.v[a:e], lr, self.betas[0], self.betas[1], self.eps,
                       self.wd, self.t, self.decoupled)

    def wait(self):
        """Order the current stream after the last update (benchmarks bracket a step with this)."""
        tr = _trainer(self.dm)
        if hasattr(tr, "wait_params"):
            tr.wait_params()

    def step(self, closure=None):
        self.t += 1
        p = self.dm.stage.params
        tr = _trainer(self.dm)
        if hasattr(tr, "settle_grads"):
            tr.settle_grads()                  # (a step without a backward since zero_grad(): lazily-zeroed matrices get their zeros)
        if not getattr(tr, "overlap_ok", False) or not p.flat.is_cuda or os.environ.get("TL_ADAM_OVERLAP", "0") != "1":
            self._update(0, p.numel)
            return
        tr.overlap_ok = False
        if self.side is None:
            self.side = torch.cuda.Stream(device=p.device)
        main = torch.cuda.current_stream()
        spans = []                                     # [a, e) of every layer in the arena, in finalisation order
        covered = []
        for j in tr.final_order:
            li = tr.layer_ids[j]
            names = [n for n in p.offsets if n.startswith(f"l{li}.")]
            a = min(p.offsets[n][0] for n in names)
            e = max(p.offsets[n][0] + (p.offsets[n][1] + 127) // 128 * 128 for n in names)
            spans.append((j, a, e))
            covered.append((a, e))
        with torch.cuda.stream(self.side):
            for j, a, e in spans:
                self.side.wait_event(tr.layer_events[j])
                self._update(a, e)
        # whatever is not a decoder layer (embedding, final norm, lm_head): final once the main stream gets here
        covered.sort()
        rest, cur = [], 0
        for a, e in covered:
            if a > cur:
                rest.append((cur, a))
            cur = max(cur, e)
        if cur < p.numel:
            rest.append((cur, p.numel))
        if rest:
            here = torch.cuda.Event()
            here.record(main)
            with torch.cuda.stream(self.side):
                self.side.wait_event(here)
                for a, e in rest:
                    self._update(a, e)
        done = torch.cuda.Event()
        done.record(self.side)
        main.wait_event(done)          # whatever the caller enqueues next sees the updated parameters
