"""``DistributedWorker`` — the reference's worker-side shard executor surface over the H100 stage.

Mirrors the handler names and argument meaning of /root/reference/tensorlink/ml/worker.py so that code written
against the reference's worker (its network process, or tests that drive a worker directly) can hold this object:

    load_module(module_info)                       :452-505  (+ _load_grouped_layers :640-715)
    _handle_forward(module_id, key, *payload)      :297-357
    _handle_backward(module_id, tag, grad)         :233-295
    _handle_generate(module_id, *payload, stream)  :359-441
    handle_forward_frame(module_id, key, bytes)    the same forward in the reference's wire format (p2p/wire.py)
    process_state_update(module_id, (op, arg))     :1268-1347

What differs: payloads are device tensors / dicts handed in and returned directly (the reference pulls pickled bytes
out of POSIX shared memory and answers through an IPC queue, `get_from_shared_memory` :303, `send_request` :349);
there is no polling `main_loop` (:1349-1437) because nothing arrives over a socket; errors raise.
`module_info` uses the reference's plan-entry keys (``module_id``, ``name``, ``type``, ``layer_range``, ``training``,
``optimizer_type`` ... ml/graphing.py:44-55).
"""
from __future__ import annotations

from typing import Any, Dict, Optional, Tuple

import torch

from .. import native as nat
from .configs import ShardModelConfig, get_config
from .stage import CudaStage


class DistributedWorker:
    def __init__(self, device: Optional[str] = None, max_batch: int = 8, max_seq: int = 4096, seed: int = 1234):
        nat.require_device()
        self.device = torch.device(device or f"cuda:{torch.cuda.current_device()}")
        self.max_batch, self.max_seq, self.seed = max_batch, max_seq, seed
        self.modules: Dict[str, CudaStage] = {}
        self.optimizers: Dict[str, Any] = {}
        self.terminate = False

    # ------------------------------------------------------------------------------------------ load
    def load_module(self, module_info: dict) -> str:
        """worker.py:452-505 / :640-715.  ``layer_range`` (a, b) inclusive selects the decoder layers of this shard;
        ``has_embed`` / ``has_head`` (extensions) place the host-side modules of the reference on this worker too."""
        module_id = module_info.get("module_id")
        if module_id is None:
            raise ValueError("For standard loading, module_id must be provided")          # same message as :468
        cfg = module_info.get("config")
        if not isinstance(cfg, ShardModelConfig):
            cfg = get_config(module_info["name"])
        if module_info.get("type", "offloaded_group") == "offloaded_group":
            a, b = module_info["layer_range"]
            layers = list(range(a, b + 1))
        else:
            layers = list(range(cfg.n_layers))
        st = CudaStage(cfg, layers, bool(module_info.get("has_embed", False)), bool(module_info.get("has_head", False)),
                       self.device, module_info.get("max_batch", self.max_batch), module_info.get("max_seq", self.max_seq),
                       n_slots=1, training=bool(module_info.get("training", False)),
                       state_dict=module_info.get("state_dict"), seed=module_info.get("seed", self.seed))
        st.n_batch = 0
        self.modules[module_id] = st
        return module_id

    # ------------------------------------------------------------------------------------------ forward / backward
    def _handle_forward(self, module_id: str, key: Tuple[int, int, str], kwargs: dict) -> dict:
        """worker.py:297-357.  ``kwargs`` = the loop live-ins; only ``hidden_states`` (and ``past_len`` for cached
        inference) are consumed, the rest is echoed back like ``LayerGroupModule`` does (injector.py:252-260)."""
        st = self.modules[module_id]
        hs = kwargs["hidden_states"].to(self.device)
        out = dict(kwargs)
        past_len = self._past_len_from_live_ins(st, kwargs, hs)
        if st.supports_training:
            from .train import StageTrainer
            if st.trainer is None:
                st.trainer = StageTrainer(st)
            out["hidden_states"] = st.trainer.forward_layers(key, hs)          # intermediates keyed like :337-341
            st.n_batch += 1
        else:
            out["hidden_states"] = st.prefill(hs, past_len, 0).clone()
        return out

    @staticmethod
    def _past_len_from_live_ins(st: CudaStage, kwargs: dict, hs: torch.Tensor) -> int:
        """Where this call's tokens start in the sequence.  A reference peer never sends ``past_len``: it ships the HF
        loop live-ins (injector.py:508-556) — ``cache_position`` [S], ``position_ids`` [B,S], ``past_key_values`` (the
        whole cache, utils.py:599-605) and the 4-D mask.  The KV cache of this stage is RESIDENT, so the position is
        taken from ``cache_position[0]`` / ``position_ids[:,0]`` and checked against what the stage has cached; inputs
        this executor cannot honour (padding masks, ragged positions, a shipped cache that disagrees with the resident
        one) raise instead of computing something else."""
        B, S = hs.shape[0], hs.shape[1]
        cand = []
        if kwargs.get("past_len") is not None:
            cand.append(int(kwargs["past_len"]))
        cp = kwargs.get("cache_position")
        if isinstance(cp, torch.Tensor) and cp.numel():
            cp = cp.reshape(-1).cpu()
            if cp.numel() != S or not torch.equal(cp, torch.arange(int(cp[0]), int(cp[0]) + S)):
                raise ValueError("cache_position must be S consecutive positions")
            cand.append(int(cp[0]))
        pid = kwargs.get("position_ids")
        if isinstance(pid, torch.Tensor) and pid.numel():
            pid = pid.reshape(-1, S).cpu()
            if not torch.equal(pid, pid[:1].expand_as(pid)) or not torch.equal(pid[0], torch.arange(int(pid[0, 0]), int(pid[0, 0]) + S)):
                raise NotImplementedError("per-row / non-consecutive position_ids (left-padded batches) are not supported by the "
                                          "wire bridge; use DistributedModel.generate(attention_mask=...) on the box instead")
            cand.append(int(pid[0, 0]))
        if cand and any(c != cand[0] for c in cand):
            raise ValueError(f"past_len / cache_position / position_ids disagree: {cand}")
        past_len = cand[0] if cand else 0
        am = kwargs.get("attention_mask")
        if isinstance(am, torch.Tensor) and am.numel():
            a = am.detach().cpu()
            if a.dim() == 2:
                trivial = bool((a != 0).all())
            else:                                    # HF's additive 4-D mask: causal = zeros on and below the diagonal
                q = a.shape[-2]
                ref = torch.ones(q, a.shape[-1], dtype=torch.bool).tril(a.shape[-1] - q)
                trivial = bool(((a == 0) == ref).all())
            if not trivial:
                raise NotImplementedError("padding / custom attention masks are not supported by the wire bridge (the stage applies the causal mask itself)")
        pkv = kwargs.get("past_key_values")
        shipped = None
        if isinstance(pkv, dict) and pkv.get("__dynamic_cache__"):
            ks = pkv.get("key_cache") or []
            shipped = int(ks[0].shape[-2]) if len(ks) and isinstance(ks[0], torch.Tensor) and ks[0].numel() else 0
        if shipped is not None and shipped not in (0, past_len):
            raise ValueError(f"shipped past_key_values hold {shipped} positions but the call starts at {past_len}")
        if past_len and not st.supports_training:
            cached = int(st.slots[0].pos_dev.item())
            if cached != past_len:
                raise ValueError(f"call starts at position {past_len} but this stage has {cached} positions cached "
                                 "(the KV cache is resident on the stage; it is not rebuilt from a shipped cache)")
        return past_len

    def handle_forward_frame(self, module_id: str, key: Tuple[int, int, str], data: bytes) -> bytes:
        """The same call in the reference's WIRE format (SURVEY.md §8 f-4): ``data`` is what the reference user side
        puts in shared memory for ``send_forward`` (ml/module.py:1549-1556: 8-byte length, args frame, kwargs frame);
        the return value is the frame its ``check_forward`` poll reads back (ml/worker.py:344-346).  A reference peer's
        node process can hand the bytes over unchanged; everything between the two frames runs on the device."""
        from ..p2p import wire
        _args, kwargs = wire.unpack_forward(data, device=self.device)
        if "hidden_states" not in kwargs:
            raise KeyError("forward request carries no hidden_states (a layer-group shard consumes kwargs only, "
                           "ml/worker.py:332-335)")
        out = self._handle_forward(module_id, key, kwargs)
        return wire.encode({k: (v.detach() if isinstance(v, torch.Tensor) else v) for k, v in out.items()})

    def handle_backward_frame(self, module_id: str, tag: Tuple[int, int, str], data: bytes) -> bytes:
        """Backward in the reference's wire format: ``data`` = one frame holding the gradient of this shard's output
        (ml/module.py:482-488 -> ml/worker.py:243-246); returns one frame holding the gradient of its input
        (ml/worker.py:289-291)."""
        from ..p2p import wire
        grad = wire.decode(data, device=self.device)
        if isinstance(grad, (tuple, list)):
            grad = grad[0]
        if not isinstance(grad, torch.Tensor):
            raise TypeError("backward request does not hold a gradient tensor")
        return wire.encode(self._handle_backward(module_id, tuple(tag), grad.to(torch.bfloat16)))

    def _handle_backward(self, module_id: str, tag: Tuple[int, int, str], loss_relay: torch.Tensor) -> torch.Tensor:
        """worker.py:233-295: backward through the shard for the micro-batch ``tag``; returns d(loss)/d(shard input)."""
        st = self.modules[module_id]
        if st.trainer is None or tag not in st.trainer.ctx:
            raise KeyError(f"no stored forward for tag {tag!r} (worker.py:253 pops intermediates[tag])")
        dx = st.trainer.backward_layers(tag, loss_relay.to(self.device))
        return dx

    # ------------------------------------------------------------------------------------------ generate
    @torch.no_grad()
    def _handle_generate(self, module_id: str, input_ids: torch.Tensor, max_new_tokens: int = 20, stream=None) -> torch.Tensor:
        """worker.py:359-441 (whole model on this worker): greedy generation; ``stream.put(token_column)`` per step
        replaces the TOKEN packets of ``TensorlinkWorkerStreamer`` (:123-144)."""
        st = self.modules[module_id]
        if not (st.has_embed and st.has_head):
            raise ValueError("generate needs a module loaded with has_embed=True and has_head=True (entire model)")
        B, S = input_ids.shape
        if B > st.max_batch or S + max_new_tokens > st.max_seq:
            raise ValueError(f"module sized for batch<={st.max_batch}, T<={st.max_seq}; got batch {B}, "
                             f"{S} prompt + {max_new_tokens} new tokens")
        ids = input_ids.to(self.device)
        x = st.prefill(st.embed(ids), 0, 0)
        st.head_argmax(x[:, -1, :].contiguous(), st.ids_dec[0][:B])
        out = [ids]
        for step in range(max_new_tokens):
            col = st.ids_dec[0][:B].clone()
            out.append(col[:, None])
            if stream is not None:
                stream.put(col.cpu())
            if step + 1 < max_new_tokens:
                st.decode(0, B)
        if stream is not None:
            stream.end()
        return torch.cat(out, dim=1)

    # ------------------------------------------------------------------------------------------ optimizer
    def process_state_update(self, module_id: str, state_update: Tuple[str, Any]) -> str:
        """worker.py:1268-1347: ("init", spec) / ("step", closure) / ("zero_grad", _) -> "loaded" / "stepped" / "zeroed"."""
        op, arg = state_update
        st = self.modules[module_id]
        if op == "init":
            kw = dict(arg or {})
            kw.pop("optimizer_type", None)
            self.optimizers[module_id] = _WorkerAdam(st, **kw)
            return "loaded"
        if op == "step":
            st.trainer.finish_backward()
            self.optimizers[module_id].step()
            return "stepped"
        if op == "zero_grad":
            if st.trainer is not None:
                st.trainer.zero_grad()
            else:
                st.params.grad.zero_()
            return "zeroed"
        raise ValueError(f"unknown optimizer op {op!r}")


class _WorkerAdam:
    def __init__(self, st: CudaStage, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.0,
                 decoupled: bool = False, **_):
        p = st.params
        self.p, self.lr, self.betas, self.eps, self.wd, self.decoupled = p, lr, betas, eps, weight_decay, decoupled
        self.m = torch.zeros(p.numel, dtype=torch.float32, device=p.device)
        self.v = torch.zeros_like(self.m)
        self.t = 0

    def step(self):
        self.t += 1
        nat.adamw_step(self.p.flat, self.p.grad, self.m, self.v, self.lr, self.betas[0], self.betas[1], self.eps, self.wd,
                       self.t, self.decoupled)
