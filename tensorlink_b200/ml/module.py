"""``DistributedModel`` — the reference's user-facing front end, driving H100 pipeline stages.

Mirrors /root/reference/tensorlink/ml/module.py: constructor signature (:251-265), ``forward`` returning an HF-style
output with ``.logits`` / ``.loss`` (:348-407), ``generate`` (:763-769), ``create_optimizer`` (:1016-1021),
``train/eval`` (:534-566), ``parameters`` (:577-650), ``distribute_model(config)`` (:699).  The reference is
hub-and-spoke: the user process RPCs each worker in turn over TCP and polls.  Here every pipeline stage is one
process on one GPU (``torchrun``), all of them construct the same ``DistributedModel`` (SPMD) and activations
go stage -> stage directly over NVLink (p2p/link.py).  With one process the whole model is a single stage.

Documented deviations from the reference: errors raise instead of being swallowed into ``{"error": ...}`` dicts
(module.py:978-985); ``dtype`` defaults to bf16 (the only dtype the sm_90a kernels implement); logits live on
the last stage (pass ``gather_logits=True`` to copy them to rank 0).
"""
from __future__ import annotations

import numbers
import os

import time
from dataclasses import dataclass, replace
from typing import Any, Callable, Dict, Optional, Union

import torch

from ..native import LP_MAX_EOS, PL_MAX_DRAFT, PL_MAX_EOS
from ..p2p.link import StageLink, init_process_group_from_env
from . import fp8 as F8
from . import graphing
from .configs import ShardModelConfig, check_moe, get_config, moe_fields


@dataclass
class CausalLMOutput:
    """The two fields of HF ``CausalLMOutputWithPast`` the reference's callers read."""
    loss: Optional[torch.Tensor] = None
    logits: Optional[torch.Tensor] = None

    def __getitem__(self, k):
        return getattr(self, k)


def _default_stage_factory(**kw):
    from .stage import CudaStage          # imports the CUDA library; raises without it
    return CudaStage(**kw)


def _config_from_hf(model) -> ShardModelConfig:
    c = model.config
    qk_norm = c.__class__.__name__.startswith("Qwen3")
    moe = moe_fields(getattr(c, "model_type", ""), lambda k: getattr(c, k, None))
    hd = getattr(c, "head_dim", None) or c.hidden_size // c.num_attention_heads
    rp = getattr(c, "rope_parameters", None) or {}
    theta = rp.get("rope_theta", getattr(c, "rope_theta", 1e6))
    return ShardModelConfig(getattr(c, "name_or_path", "") or c.__class__.__name__, c.hidden_size,
                            c.intermediate_size, c.num_hidden_layers, c.num_attention_heads,
                            c.num_key_value_heads, hd, c.vocab_size, tied=bool(c.tie_word_embeddings),
                            qkv_bias=not qk_norm, qk_norm=qk_norm, rope_theta=float(theta),
                            rms_eps=float(c.rms_norm_eps), max_pos=int(c.max_position_embeddings), **moe)


# HF forward / generate keywords that change nothing here when left at these values (anything else raises instead of
# being dropped silently: the reference forwards every keyword to HF, module.py:763-769)
_NEUTRAL_KW = {"use_cache": (True, False, None), "return_dict": (True, None), "output_attentions": (False, None),
               "output_hidden_states": (False, None), "num_beams": (1, None), "num_return_sequences": (1, None),
               "repetition_penalty": (1.0, None), "past_key_values": (None,), "position_ids": (None,),
               "return_dict_in_generate": (False, None), "logits_to_keep": (0, None), "min_new_tokens": (0, None),
               # assisted decoding drafts a fixed K per captured verify step: no schedule, no confidence cut
               "num_assistant_tokens_schedule": ("constant", None), "assistant_confidence_threshold": (None,)}


def _warpers(min_p=None, typical_p=None, epsilon_cutoff=None, eta_cutoff=None) -> dict:
    """The sampling dict's entries for HF's MinP / Typical / Epsilon / Eta warpers (ml/stage.py WARPER_KEYS), active
    ones only: as in HF's ``_get_logits_processor``, min_p is off at None or 0, typical_p at None or >= 1, and
    epsilon_cutoff / eta_cutoff at None or outside (0, 1); the values HF's warpers reject raise ValueError."""
    out = {}
    if min_p is not None:
        if not 0.0 <= float(min_p) <= 1.0:
            raise ValueError(f"`min_p` has to be a float in the [0, 1] interval, but is {min_p}")
        if float(min_p) > 0.0:
            out["min_p"] = float(min_p)
    if typical_p is not None and float(typical_p) < 1.0:
        if not float(typical_p) > 0.0:
            raise ValueError(f"`typical_p` has to be a float > 0 and < 1, but is {typical_p}")
        out["typical_p"] = float(typical_p)
    for name, key, v in (("epsilon_cutoff", "epsilon", epsilon_cutoff), ("eta_cutoff", "eta", eta_cutoff)):
        if v is not None and 0.0 < float(v) < 1.0:
            out[key] = float(v)
    return out


def _check_unconsumed(kwargs: dict, what: str):
    for k, v in kwargs.items():
        ok = _NEUTRAL_KW.get(k)
        if ok is None or not any(v is o or (o is not None and v == o) for o in ok):
            raise NotImplementedError(f"{what}: keyword {k}={v!r} is not supported by the H100 stage executor "
                                      "(it would be silently ignored otherwise)")


# What a generate call may need of its stage, each with the attribute that provides it.  The CUDA stage provides all
# of them; another stage (the CPU stages of the tests) provides those whose attribute it has.
_STAGE_FEATURES = {"scores": "set_score_log", "sampling": "set_sampling", "processors": "set_logits_processors",
                   "drafts": "prompt_lookup_begin", "kv_start": "supports_kv_start", "check": "check"}


def _stage_supports(stage, feature: str, what: Optional[str] = None) -> bool:
    """Whether ``stage`` provides ``feature`` (a key of _STAGE_FEATURES).  With ``what``, a stage without it raises
    NotImplementedError("<what> needs the CUDA stage")."""
    from .stage import CudaStage
    ok = isinstance(stage, CudaStage) or bool(getattr(stage, _STAGE_FEATURES[feature], False))
    if not ok and what is not None:
        raise NotImplementedError(f"{what} needs the CUDA stage")
    return ok


def _logits_processors(repetition_penalty=None, no_repeat_ngram_size=None, min_new_tokens=None,
                       eos_token_id=None) -> Optional[dict]:
    """HF's ``repetition_penalty`` / ``no_repeat_ngram_size`` / ``min_new_tokens`` as {penalty, ngram, min_new, eos}, or
    None when every one is at its neutral value (1.0 / 0 / 0, or None).  ``eos`` lists the EOS ids ``min_new_tokens``
    holds back (empty without it or without ``eos_token_id``, where HF's processor is a no-op).  Invalid values raise
    ValueError, as HF does; more EOS ids than the device parameter block holds raise NotImplementedError."""
    p = 1.0 if repetition_penalty is None else repetition_penalty
    if isinstance(p, bool) or not isinstance(p, numbers.Real) or not p > 0:
        raise ValueError(f"repetition_penalty has to be a strictly positive float, but is {repetition_penalty!r}")
    n, k = (0 if v is None else v for v in (no_repeat_ngram_size, min_new_tokens))
    for name, v in (("no_repeat_ngram_size", n), ("min_new_tokens", k)):
        if isinstance(v, bool) or not isinstance(v, numbers.Integral) or v < 0:
            raise ValueError(f"{name} has to be a non-negative integer, but is {v!r}")
    if p == 1.0 and n == 0 and k == 0:
        return None
    eos = _eos_list(eos_token_id) if k > 0 else []
    if len(eos) > LP_MAX_EOS:
        raise NotImplementedError(f"min_new_tokens with {len(eos)} EOS ids (at most {LP_MAX_EOS})")
    return {"penalty": float(p), "ngram": int(n), "min_new": int(k), "eos": eos}


def _prompt_lookup(num_tokens, ngram, shape, max_new, max_seq, sampling=None, procs=None, world=1, stage=None,
                   eos_token_id=None) -> Optional[dict]:
    """HF's ``prompt_lookup_num_tokens`` / ``max_matching_ngram_size`` as {K, ngram}, or None when prompt lookup is off
    (``num_tokens`` None).  ``shape``: the [rows, S] of the prompt that reaches the cache.  Values HF rejects, more than
    PL_MAX_DRAFT drafts, more than one row, or a cache too short for the last verify step raise ValueError; what the
    verify step does not implement (logits processors, several stages, another stage than the CUDA one, more EOS ids
    than the device parameter block holds) raises NotImplementedError.  ``sampling`` (do_sample) is accepted."""
    if num_tokens is None:
        return None
    n = 2 if ngram is None else ngram
    for name, v in (("prompt_lookup_num_tokens", num_tokens), ("max_matching_ngram_size", n)):
        if isinstance(v, bool) or not isinstance(v, numbers.Integral) or v < 1:
            raise ValueError(f"{name} has to be a positive integer, but is {v!r}")
    K = int(num_tokens)
    if K > PL_MAX_DRAFT:
        raise ValueError(f"prompt_lookup_num_tokens={K}: a verify step runs at most {PL_MAX_DRAFT} drafts")
    rows, S = shape
    if rows != 1:
        raise ValueError(f"prompt lookup decoding generates one row at a time, got {rows} rows")
    if S + max_new + K > max_seq:
        raise ValueError(f"prompt lookup needs S + max_new_tokens + prompt_lookup_num_tokens <= max_seq (the last verify "
                         f"step writes K+1 cache slots); got {S} + {max_new} + {K} > {max_seq}")
    if procs is not None:
        raise NotImplementedError("prompt_lookup_num_tokens with repetition_penalty / no_repeat_ngram_size / min_new_tokens")
    if world > 1:
        raise NotImplementedError("prompt_lookup_num_tokens on a pipeline of more than one stage")
    if len(_eos_list(eos_token_id)) > PL_MAX_EOS:
        raise NotImplementedError(f"prompt_lookup_num_tokens with more than {PL_MAX_EOS} EOS ids")
    _stage_supports(stage, "drafts", f"prompt_lookup_num_tokens{' with do_sample=True' if sampling is not None else ''}")
    return {"K": K, "ngram": int(n)}


# num_assistant_tokens when the keyword is absent: the K with the most expected tokens per ms in tools/bench_assisted.py
# (Qwen2.5-7B target, Qwen2.5-0.5B assistant, one H100), with an ASSUMED agreement of 0.8 per draft token between the two
# models.  The same rule on sampled round costs (``--sampled``) also gives 2, so the default serves do_sample as well.  It
# changes speed only: never the greedy output, nor the distribution of the sampled one.
ASSISTED_DEFAULT_K = 2


def _device_key(d):
    """(type, index) of a device, "cuda" meaning the current CUDA device."""
    d = torch.device(d)
    return d.type, (torch.cuda.current_device() if d.type == "cuda" and d.index is None else d.index)


def _assisted(target, assistant, num_tokens, shape, max_new, sampling=None, procs=None) -> dict:
    """HF's ``assistant_model`` / ``num_assistant_tokens`` as {K, ngram, assistant (its stage)}.  A non-DistributedModel
    raises TypeError; the target as its own assistant, a bad K (1..PL_MAX_DRAFT), more than one row or a cache of either
    model too short for the last verify step raise ValueError; what the verify step does not implement (logits
    processors, several stages on either side, a stage other than the CUDA one, an assistant on another device) raises
    NotImplementedError.  ``sampling`` (do_sample) is accepted."""
    if not isinstance(assistant, DistributedModel):
        raise TypeError(f"assistant_model has to be a DistributedModel, got {type(assistant).__name__}; wrap an HF "
                        "module as DistributedModel(hf_model, training=False)")
    if assistant is target:
        raise ValueError("assistant_model is the model itself (the two would share one KV cache)")
    K = ASSISTED_DEFAULT_K if num_tokens is None else num_tokens
    if isinstance(K, bool) or not isinstance(K, numbers.Integral) or not 1 <= K <= PL_MAX_DRAFT:
        raise ValueError(f"num_assistant_tokens has to be an integer in 1..{PL_MAX_DRAFT} (a verify step runs at most "
                         f"{PL_MAX_DRAFT} drafts), but is {num_tokens!r}")
    K = int(K)
    rows, S = shape
    if rows != 1:
        raise ValueError(f"assisted decoding generates one row at a time, got {rows} rows")
    for who, m in (("the model", target), ("the assistant", assistant)):
        if S + max_new + K > m.max_seq:
            raise ValueError(f"assisted decoding needs S + max_new_tokens + num_assistant_tokens <= max_seq of {who} (the "
                             f"last verify step writes K+1 cache slots); got {S} + {max_new} + {K} > {m.max_seq}")
    if procs is not None:
        raise NotImplementedError("assistant_model with repetition_penalty / no_repeat_ngram_size / min_new_tokens")
    if target.world > 1 or assistant.world > 1:
        raise NotImplementedError("assistant_model with a model or an assistant on a pipeline of more than one stage")
    for st in (target.stage, assistant.stage):
        _stage_supports(st, "drafts", f"assistant_model{' with do_sample=True' if sampling is not None else ''}")
    if _device_key(assistant.stage.device) != _device_key(target.stage.device):
        raise NotImplementedError(f"assistant_model on {assistant.stage.device} for a model on {target.stage.device} "
                                  "(both run on one device)")
    return {"K": K, "ngram": 0, "assistant": assistant.stage}


def _check_attention_mask(mask, shape):
    """forward(): only the all-ones mask (no padding) is accepted; a mask with zeros means padded prompts, whose rows
    would otherwise attend to pad tokens at shifted positions.  (``generate`` handles left-padded batches.)"""
    if mask is None:
        return
    if tuple(mask.shape) != tuple(shape):
        raise ValueError(f"attention_mask shape {tuple(mask.shape)} != input_ids shape {tuple(shape)}")
    if not bool((mask != 0).all()):
        raise NotImplementedError("padded rows (attention_mask with zeros) are not supported by forward(): pass rows of "
                                  "equal length")


def _train_mask(mask, shape):
    """A training batch's ``attention_mask`` as (kv_start, real): ``kv_start[b]`` is the number of leading pad tokens of
    row b and ``real`` (bool [B,S], on the host) marks its real tokens; None when the mask has no zero.  Each row's ones
    must form one run of at least one token (left, right or both sides padded): holes raise NotImplementedError, an
    empty row or a mask shaped unlike ``input_ids`` raises ValueError."""
    if mask is None:
        return None
    if tuple(mask.shape) != tuple(shape):
        raise ValueError(f"attention_mask shape {tuple(mask.shape)} != input_ids shape {tuple(shape)}")
    real = (mask != 0).cpu()
    if bool(real.all()):
        return None
    lengths = real.sum(1)
    if int(lengths.min()) == 0:
        raise ValueError("attention_mask has a row without any real token")
    starts = real.long().argmax(1)
    cols = torch.arange(real.shape[1])[None, :]
    if not torch.equal(real, (cols >= starts[:, None]) & (cols < (starts + lengths)[:, None])):
        raise NotImplementedError("attention_mask rows must be one run of ones (padding on the left and/or the right, "
                                  "no holes)")
    return [int(v) for v in starts.tolist()], real


def _left_pad_groups(mask: torch.Tensor):
    """A left-padded batch (HF's convention for generation: ``tokenizer(..., padding=True, padding_side='left')``)
    as {real length: [row indices]}; None when no row is padded.  Right padding / holes raise."""
    m = (mask != 0).cpu()
    if bool(m.all()):
        return None
    S = m.shape[1]
    lengths = m.sum(1)
    want = torch.arange(S)[None, :] >= (S - lengths)[:, None]           # zeros, then ones
    if not torch.equal(m, want) or int(lengths.min()) == 0:
        raise NotImplementedError("attention_mask must describe LEFT-padded prompts (zeros, then ones; at least one token per row)")
    groups = {}
    for r, L in enumerate(lengths.tolist()):
        groups.setdefault(int(L), []).append(r)
    return groups


def _left_pad_starts(mask: torch.Tensor):
    """A left-padded batch as (trim, starts): ``trim`` leading columns are pad in every row and are dropped, and row b of
    the remaining ``S - trim`` columns starts with ``starts[b]`` pad slots.  None when no row is padded; right padding /
    holes raise (``_left_pad_groups``)."""
    if _left_pad_groups(mask) is None:
        return None
    lengths = (mask != 0).sum(1).cpu()
    width = int(lengths.max())
    return mask.shape[1] - width, [width - int(L) for L in lengths.tolist()]


EOS_CHECK_EVERY = 16       # decode steps between two host-side "has every row emitted EOS?" checks


def _output_flags(return_dict_in_generate=None, output_scores=None, output_logits=None) -> Optional[dict]:
    """HF's ``return_dict_in_generate`` / ``output_scores`` / ``output_logits`` as {scores, logits} (what to log), or
    None when the plain tensor is returned.  Each accepts True, False or None; without ``return_dict_in_generate=True``
    the other two are ignored, as HF ignores them."""
    for name, v in (("return_dict_in_generate", return_dict_in_generate), ("output_scores", output_scores),
                    ("output_logits", output_logits)):
        if v is not None and not isinstance(v, bool):
            raise ValueError(f"{name} has to be True, False or None, but is {v!r}")
    if not return_dict_in_generate:
        return None
    return {"scores": bool(output_scores), "logits": bool(output_logits)}


def _eos_list(eos_token_id):
    if eos_token_id is None:
        return []
    if isinstance(eos_token_id, torch.Tensor):              # HF accepts an int, a list or a tensor of ids
        return [int(e) for e in eos_token_id.reshape(-1).tolist()]
    return [int(e) for e in eos_token_id] if isinstance(eos_token_id, (list, tuple)) else [int(eos_token_id)]


@dataclass(frozen=True)
class _Request:
    """One ``generate`` call, parsed once (``DistributedModel._request``) and the same on every rank."""
    max_new: int
    shape: tuple                      # [rows, S] of the prompt the run sees (from the first rank, as those below)
    sampling: Optional[dict] = None   # {temperature, top_k, top_p, seed, + active warpers}, or None: greedy
    eos: tuple = ()                   # the EOS ids
    pad_token_id: Optional[int] = None
    procs: Optional[dict] = None      # _logits_processors
    draft: Optional[dict] = None      # the draft source: _prompt_lookup or _assisted, or None
    out: Optional[dict] = None        # _output_flags
    streamer: Any = None
    use_graph: bool = True
    profile: bool = False
    # a left-padded batch either as the leading columns that are pad in every row (dropped before the run, back in the
    # result) and the per-row key starts of the rest, or, on a stage without per-row key starts, as {real length:
    # [rows]}; and the logits processors' starting history
    pad_cols: Optional[torch.Tensor] = None
    kv_start: Optional[list] = None
    groups: Optional[dict] = None
    history: Optional[torch.Tensor] = None


def _all_rows_finished(tokens: torch.Tensor, eos_ids) -> bool:
    """tokens [rows, cols] generated so far: True once every row holds an EOS (one small device reduction + sync)."""
    hit = torch.zeros_like(tokens, dtype=torch.bool)
    for e in eos_ids:
        hit |= tokens == e
    return bool(hit.any(1).all().item())


def apply_eos(result: torch.Tensor, prompt_len: int, eos_token_id=None, pad_token_id=None) -> torch.Tensor:
    """HF ``generate`` stopping semantics applied to a generation [B, S+new]: everything after a row's first EOS
    becomes ``pad_token_id`` (default: the EOS id) and the result ends where the last row finished.  (The decode loop
    checks every ``EOS_CHECK_EVERY`` steps whether all rows are finished and stops computing then; the at most 15 surplus
    columns are cut here.)"""
    if eos_token_id is None:
        return result
    eos_ids = _eos_list(eos_token_id)
    pad = eos_ids[0] if pad_token_id is None else int(pad_token_id)
    new = result[:, prompt_len:]
    if new.shape[1] == 0:
        return result
    is_eos = torch.zeros_like(new, dtype=torch.bool)
    for e in eos_ids:
        is_eos |= new == e
    seen_before = (is_eos.cumsum(1) - is_eos.long()) > 0
    new = torch.where(seen_before, torch.full_like(new, pad), new)
    first = torch.where(is_eos.any(1), is_eos.long().argmax(1) + 1, torch.full_like(new[:, 0], new.shape[1]))
    return torch.cat([result[:, :prompt_len], new[:, :int(first.max())]], dim=1)


class DistributedModel(torch.nn.Module):
    def __init__(self, model: Union[torch.nn.Module, str, ShardModelConfig], n_pipelines: int = 1,
                 optimizer=None, scheduler_type=None, device: Optional[str] = None,
                 dtype: torch.dtype = torch.bfloat16, trusted: bool = False, node: Optional[Any] = None,
                 training: bool = True, verbose: bool = False, tokenizer=None, config: Optional[dict] = None,
                 *, max_batch: int = 8, max_seq: int = 4096, seed: int = 1234, init: str = "seeded",
                 balanced_plan: bool = False, link: Optional[StageLink] = None, max_tokens: Optional[int] = None,
                 quantization_config=None, _stage_factory: Optional[Callable] = None):
        """``model``: an HF Qwen2 / Qwen3 module, a ShardModelConfig or registered config name (weights drawn by
        ``init``: "seeded" or "device"), or a local HF checkpoint directory, bf16 or in HF's fine-grained FP8 layout
        (``quantization_config.quant_method == "fp8"``, e4m3, 128x128 blocks; each stage reads its own ``weight`` and
        ``weight_scale_inv`` tensors).

        ``quantization_config``: HF's ``FineGrainedFP8Config`` or the same dict.  It quantizes the decoder layers'
        Linears of an in-memory bf16 model on load with HF's rule (``Fp8Quantize``).  FP8 models run weight-only (W8A16):
        each weight is bf16(float32(w) * scale_inv[block]), so their outputs equal, bit for bit, those of the bf16 model
        over HF's dequantized weights (``FineGrainedFP8Config(dequantize=True)``).  HF's GPU ``FP8Linear`` also
        quantizes the activations per 1x128 group; that is deliberately not done here.  Norms, biases, the embedding
        and the lm_head stay bf16.  Training FP8 weights is not supported: pass ``training=False``."""
        super().__init__()
        if dtype != torch.bfloat16:
            raise NotImplementedError("tensorlink_b200 computes in bf16 with fp32 accumulation; pass dtype=torch.bfloat16")
        quantization = F8.parse_quantization_config(quantization_config)
        state_dict = None
        if isinstance(model, torch.nn.Module):
            self.cfg = _config_from_hf(model)
            state_dict = model.state_dict()
            if any(t.dtype == torch.float8_e4m3fn for t in state_dict.values()):
                # an HF module loaded with FineGrainedFP8Config: its Linears hold e4m3 codes + weight_scale_inv
                hf_q = getattr(model.config, "quantization_config", None)
                if hf_q is None:
                    raise NotImplementedError("an HF module with float8 weights but no config.quantization_config")
                quantization = F8.parse_quantization_config(hf_q)
        elif isinstance(model, ShardModelConfig):
            self.cfg = model
        elif isinstance(model, str) and os.path.isdir(model) and os.path.exists(os.path.join(model, "config.json")):
            # a local checkpoint in the HF layout: each stage reads only its own tensors (worker.py:542-638)
            from .checkpoint import LazyCheckpoint, config_from_dir, quantization_from_dir
            self.cfg = config_from_dir(model)
            quantization = quantization_from_dir(model) or quantization
            state_dict = LazyCheckpoint(model)
        else:
            self.cfg = get_config(model)
        if quantization is not None and training:
            raise NotImplementedError("training with FP8 weights is not supported: load an FP8 model with training=False")
        if self.cfg.is_moe:
            check_moe(self.cfg)
            if training:
                raise NotImplementedError("training a Qwen3-MoE model is not supported: load it with training=False")
            if quantization is not None:
                raise NotImplementedError("FP8 Qwen3-MoE weights are not supported: load the bf16 checkpoint")
        self.quantization = quantization
        self.model_name = self.cfg.name
        self.name = self.model_name
        self.tokenizer = tokenizer
        self.n_pipelines = max(1, int(n_pipelines))          # micro-batches in flight (module.py:374-399)
        self.n_datalines = 1
        self.optimizer = optimizer
        self.scheduler = scheduler_type
        self.training = training
        self.verbose = verbose
        self.trusted = trusted
        self.job_id = None
        if node is None:
            from ..nodes.nodes import User
            node = User()
        self.node = node
        self.node_requests = getattr(node, "node_requests", None)
        self.node_responses = getattr(node, "node_responses", None)
        self.mpc_lock = getattr(node, "mpc_lock", None)

        if link is None:
            init_process_group_from_env()
            link = StageLink.from_env()
        self.link = link
        self.rank, self.world = link.rank, link.world
        if device is None:
            device = f"cuda:{torch.cuda.current_device()}" if torch.cuda.is_available() else "cpu"
        self.device = torch.device(device)

        self.config = config if config else {}
        self.max_batch, self.max_seq, self.seed = max_batch, max_seq, seed
        self._stage_factory = _stage_factory or _default_stage_factory
        self._stage_kw = dict(init=init, state_dict=state_dict, balanced=balanced_plan, max_tokens=max_tokens)
        self.distributed_graph: Dict[str, Any] = {}
        self.stage = None
        self.timers: Dict[str, float] = {}
        if self.node.__class__.__name__ == "User":
            self._initialize_distribution()

    # ------------------------------------------------------------------------------------------ distribution
    def _initialize_distribution(self):
        """module.py:987-1021: obtain a plan, distribute, expose ``create_optimizer``."""
        plan = self.config or graphing.make_plan(self.cfg, self.world, self.training, self._stage_kw["balanced"])
        self.distribute_model(plan)

    def distribute_model(self, config: Optional[dict] = None):
        """module.py:699-761.  Every rank materialises exactly its entries of the plan."""
        plan = config or self.config or graphing.make_plan(self.cfg, self.world, self.training)
        if graphing.n_stages(plan) != self.world:
            raise ValueError(f"plan has {graphing.n_stages(plan)} stages but the job has {self.world} ranks")
        self.distributed_graph = plan
        layers = graphing.stage_layers(plan, self.rank)
        n_slots = self.n_pipelines
        per_slot = (self.max_batch + n_slots - 1) // n_slots
        self.stage = self._stage_factory(cfg=self.cfg, layer_ids=layers, has_embed=self.rank == 0,
                                         has_head=self.rank == self.world - 1, device=self.device,
                                         max_batch=per_slot, max_seq=self.max_seq, n_slots=n_slots,
                                         training=self.training, state_dict=self._stage_kw["state_dict"],
                                         seed=self.seed, init=self._stage_kw["init"],
                                         max_tokens=self._stage_kw["max_tokens"],
                                         **({"quantization": self.quantization} if self.quantization else {}))
        self._stage_kw["state_dict"] = None
        return plan

    # ------------------------------------------------------------------------------------------ nn.Module surface
    def train(self, mode: bool = True):
        self.training = mode
        return self

    def eval(self):
        return self.train(False)

    def parameters(self, recurse: bool = True, distributed: bool = True, load: bool = True):
        """module.py:577-650: this rank's parameters under their HF names (values, not nn.Parameters)."""
        return iter(self.stage.params.hf_state_dict().values())

    def state_dict(self, *a, gather: bool = False, **k):
        """This rank's tensors under their HF names.  ``gather=True``: the WHOLE model's state dict on the first rank, on the
        host (what the reference's ``parameters(distributed=True, load=True)`` pulls from its workers, module.py:577-650);
        the other ranks get their own part.  For checkpoints prefer ``save_pretrained`` (each stage writes its own file)."""
        sd = self.stage.params.hf_state_dict()
        if not gather or self.world == 1:
            return sd
        parts = self.link.gather_object({k_: v.detach().cpu() for k_, v in sd.items()}, 0)
        if not self.link.first:
            return sd
        whole: Dict[str, torch.Tensor] = {}
        for part in parts:
            whole.update(part)
        if self.cfg.tied and "lm_head.weight" in whole and "model.embed_tokens.weight" in whole:
            whole["lm_head.weight"] = whole["model.embed_tokens.weight"]      # one tensor under both names, like HF
        return whole

    def save_pretrained(self, path: str):
        """Write this job's weights as an HF-layout checkpoint (one safetensors file per stage + index + config)."""
        from .checkpoint import save_checkpoint
        save_checkpoint(self, path)

    def create_optimizer(self, **optimizer_kwargs):
        if self.cfg.is_moe:
            raise NotImplementedError("training a Qwen3-MoE model is not supported (no optimizer for a MoE model)")
        if self.quantization is not None:
            raise NotImplementedError("training with FP8 weights is not supported (no optimizer for an FP8 model)")
        from .optim import create_distributed_optimizer
        return create_distributed_optimizer(self, self.optimizer, **optimizer_kwargs)

    # ------------------------------------------------------------------------------------------ forward
    def forward(self, *args, **kwargs) -> CausalLMOutput:
        """One forward through every stage (module.py:348-407).  ``input_ids`` positional or keyword (:355-359).
        Inference: logits [B,S,V] on the last stage, rows of equal length only.  Training (``self.training`` with a
        grad-enabled stage): handled by ``ml/train.py``; a padded ``attention_mask`` is accepted there
        (``train_forward``)."""
        input_ids = kwargs.pop("input_ids", args[0] if args else None)
        labels = kwargs.pop("labels", None)
        gather = kwargs.pop("gather_logits", False)
        mask = kwargs.pop("attention_mask", None)
        training = self.training and getattr(self.stage, "supports_training", False)
        padding = None
        if self.link.first and input_ids is not None:
            if training:
                padding = _train_mask(mask, input_ids.shape)
            else:
                _check_attention_mask(mask, input_ids.shape)
        _check_unconsumed(kwargs, "DistributedModel.forward")
        if training:
            from .train import train_forward
            return train_forward(self, input_ids, labels, padding)
        return self._infer_forward(input_ids, gather)

    def _infer_forward(self, input_ids: Optional[torch.Tensor], gather: bool) -> CausalLMOutput:
        link, st, cfg = self.link, self.stage, self.cfg
        shape = link.broadcast_object(tuple(input_ids.shape) if link.first else None)
        B, S = shape
        # micro-batches of at most the stage's per-slot batch flow through the ranks back to back
        mb = min(B, st.max_batch)
        parts = []
        for a in range(0, B, mb):
            e = min(B, a + mb)
            if link.first:
                x = st.embed(input_ids[a:e].to(self.device))
            else:
                x = torch.empty(e - a, S, cfg.hidden, dtype=torch.bfloat16, device=self.device)
                link.recv_prev(x)
            x = st.prefill(x, 0, 0)
            if not link.last:
                link.send_next(x.clone())
            else:
                parts.append(st.head_logits(x.reshape((e - a) * S, cfg.hidden)).view(e - a, S, cfg.vocab))
        logits = torch.cat(parts, dim=0) if parts else None
        if gather and self.world > 1:
            if link.last:
                link.send_up(logits.contiguous(), 0)
            elif link.first:
                logits = torch.empty(B, S, cfg.vocab, dtype=torch.bfloat16, device=self.device)
                link.recv_up(logits, self.world - 1)
        link.flush()
        return CausalLMOutput(logits=logits)

    # ------------------------------------------------------------------------------------------ peer-memory decode
    def _peer_ring(self, n_mb: int):
        """The mailbox ring for decode hops (p2p/peer.py), or None: TL_P2P=nccl, or stages that are not on CUDA devices
        (the gloo tests drive this class with a CPU stage).  Built collectively on first use."""
        if os.environ.get("TL_P2P", "peer") == "nccl" or self.device.type != "cuda":
            return None
        if getattr(self, "_ring", None) is None:
            from ..p2p.peer import PeerRing
            st = self.stage
            self._ring = PeerRing(self.link, len(st.slots), st.max_batch, self.cfg.hidden, st.max_seq, self.device)
        return self._ring

    def _decode_ring(self, ring, input_ids, req: _Request, b, n_mb, t0):
        """Decode rounds with every hop on peer memory.  The host only enqueues: max_new-1 graph replays per
        micro-batch (wait -> layers -> store into the neighbour -> signal), no synchronisation until the end; the
        first stage logs each token column on the device (``ring.out_log``)."""
        link, st, dev = self.link, self.stage, self.device
        streamer, max_new = req.streamer, req.max_new
        B = req.shape[0]
        span = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        span[0].record()
        step_done = []
        n_cols = max_new                              # token columns that will exist when the loop ends
        for step in range(max_new):
            for m in range(n_mb):
                if step < max_new - 1:
                    st.decode(m, b, req.use_graph, ring=ring)
                elif link.first:                                   # last column: nothing left to compute
                    ring.wait_ids(m)
                    ring.log_token(m, b)
            if streamer is not None and link.first:
                ev = torch.cuda.Event()
                ev.record()
                step_done.append(ev)
            if req.eos and step < max_new - 1 and (step + 1) % EOS_CHECK_EVERY == 0:
                # HF stops once every row has emitted EOS.  Columns 0..step are logged on the first stage; all ranks
                # drain their queues (no persistent kernel is in flight during the collective) and agree on stopping.
                torch.cuda.synchronize(dev)
                flag = torch.zeros(1, dtype=torch.int32, device=dev)
                if link.first and _all_rows_finished(ring.out_log[:n_mb, :b, :step + 1].reshape(B, step + 1), req.eos):
                    flag.fill_(1)
                link.broadcast(flag, 0)
                if int(flag.item()):
                    n_cols = step + 1
                    break
        span[1].record()
        if streamer is not None and link.first:
            for step, ev in enumerate(step_done):                  # step's graph logged column `step` before its event
                ev.synchronize()
                streamer.put(ring.out_log[:n_mb, :b, step].reshape(-1).cpu())
        torch.cuda.synchronize(dev)
        ring.check()
        if req.profile:
            self.timers["decode_span_s"] = span[0].elapsed_time(span[1]) * 1e-3
            self.timers["decode_busy_s"] = self.timers["decode_span_s"] - float(ring.wait_ns.item()) * 1e-9
        tokens = ring.out_log[:n_mb, :b, :n_cols].reshape(B, n_cols) if link.first else None
        return self._finish(req, input_ids, tokens, n_cols, t0)

    def _generate_left_padded(self, input_ids, req: _Request):
        """HF semantics for a left-padded batch on a stage without per-row key starts (``supports_kv_start``): every row
        attends to its own tokens only, at positions 0..L-1.  Rows of equal real length are generated together (one
        uniform run per length: the KV cache and RoPE positions of a run start at the row's first real token, so no pad
        key exists to be masked); the result keeps HF's layout [pads | prompt | new tokens | pad_token_id...].  Sampled,
        the run of length L draws with the seed + L."""
        dev, first = self.device, self.link.first
        B, S = req.shape
        pad_id = req.pad_token_id if req.pad_token_id is not None else (req.eos[0] if req.eos else 0)
        out = torch.full((B, S + req.max_new), pad_id, dtype=torch.int64, device=dev)
        if first:
            out[:, :S] = input_ids.to(dev)
        longest = 0
        for L in sorted(req.groups):
            rows = req.groups[L]
            sub = input_ids[rows][:, S - L:].contiguous() if first else None
            sampling = None if req.sampling is None else dict(req.sampling, seed=req.sampling["seed"] + L)
            got = self._generate_batch(sub, replace(req, shape=(len(rows), L), groups=None, sampling=sampling))
            n_new = got.shape[1] - L
            out[torch.as_tensor(rows, device=dev), S:S + n_new] = got[:, L:].to(dev)
            longest = max(longest, n_new)
        out = out[:, :S + longest].contiguous()
        self.link.broadcast(out, 0)                  # every rank returns the whole result, prompt and pads included
        return out

    def _generate_lookup(self, input_ids, req: _Request):
        """Generation of one row with prompt-lookup drafts (``_prompt_lookup``) or an assistant's (``_assisted``) on the
        one CUDA stage, greedy or sampled (``req.sampling``): prefill, the first token from the head, then verify steps
        (ml/stage.py ``prompt_lookup_step``), each drafting K tokens on the device (from the row's history, or by the assistant,
        whose cache starts with the prompt's prefill) and emitting 1..K+1 tokens.  The host replays rounds of
        r = max(1, (max_new - count) // (K+1)) steps (at most EOS_CHECK_EVERY with ``eos_token_id``), so no step runs
        once max_new tokens are out, and reads the token count once per round."""
        st, dev, max_new, streamer = self.stage, self.device, req.max_new, req.streamer
        K, asst = req.draft["K"], req.draft.get("assistant")
        S = input_ids.shape[1]
        st.set_sampling(req.sampling)              # no logits processors: the plain argmax or sampling head
        if req.sampling is not None:
            st.sample_ctr.zero_()                  # a seed names ONE set of streams (ml/stage.py STREAM_PL_ROWS)
        st.set_logits_processors(None)
        t0 = time.perf_counter()
        ids = input_ids.to(dev)
        x = st.prefill(st.embed(ids), 0, 0)
        first = st.ids_dec[0][:1]
        st.head_argmax(x[:, -1, :].contiguous(), first, 0)
        steps, count = 0, 0
        tokens = torch.zeros(0, dtype=torch.int64)
        if max_new >= 1:
            if asst is not None:
                asst.prefill(asst.embed(ids), 0, 0)
            st.prompt_lookup_begin(torch.cat([ids, first.view(1, 1)], dim=1), K, req.draft["ngram"], S + max_new,
                                   list(req.eos), assistant=asst)
            while True:
                count = st.prompt_lookup_count()
                new = st.prompt_lookup_tokens(tokens.numel(), count)
                tokens = torch.cat([tokens, new])
                if streamer is not None:
                    for j in range(new.numel()):
                        streamer.put(new[j:j + 1])
                if count >= max_new or any(int(t) in req.eos for t in new):
                    break
                r = max(1, (max_new - count) // (K + 1))
                if req.eos:
                    r = min(r, EOS_CHECK_EVERY)
                for _ in range(r):
                    st.prompt_lookup_step(req.use_graph)
                steps += r
        self.timers["prompt_lookup_steps" if asst is None else "assisted_steps"] = steps
        tokens = tokens[:max_new].view(1, -1)
        return self._finish(req, ids, tokens, tokens.shape[1], t0)

    def _finish(self, req: _Request, input_ids, tokens, n_cols: int, t0: float):
        """The end of every run: the result [B, S + n_cols], the prompt then the first ``n_cols`` columns of the first
        stage's ``tokens``, on every rank; the stage's error check; HF's EOS cut (``apply_eos``); the streamer's end;
        ``timers["generate_wall_s"]``.  With ``req.out``, returns (result, logs): the last stage's score logs of the
        generated columns the cut kept, on every rank, as {"scores" / "logits": a tuple of fp32 [B, V] tensors}."""
        link, dev = self.link, self.device
        B, S = req.shape
        if link.first:
            result = torch.cat([input_ids.to(dev), tokens[:, :n_cols].to(dev)], dim=1)
        else:
            result = torch.empty(B, S + n_cols, dtype=torch.int64, device=dev)
        link.broadcast(result, 0)
        if _stage_supports(self.stage, "check"):
            self.stage.check()
        if req.streamer is not None and link.first:
            req.streamer.end()
        self.timers["generate_wall_s"] = time.perf_counter() - t0
        result = apply_eos(result, S, list(req.eos) or None, req.pad_token_id)
        logs, n_new = {}, result.shape[1] - S
        for kind in ("scores", "logits"):
            if req.out is None or not req.out[kind]:
                continue
            if link.last:
                t = self.stage.score_log_copy(kind, B, n_new)
            else:
                t = torch.empty(n_new, B, self.cfg.vocab, dtype=torch.float32, device=dev)
            link.broadcast(t, self.world - 1)
            logs[kind] = tuple(t.unbind(0))
        return result if req.out is None else (result, logs)

    # ------------------------------------------------------------------------------------------ generate
    @torch.no_grad()
    def generate(self, *args, **kwargs) -> Optional[torch.Tensor]:
        """Generation (module.py:763-769 delegates to HF ``generate``).  Greedy by default; ``do_sample=True`` draws every
        token on the last stage's GPU from the distribution HF's warpers define — ``temperature`` (default 1.0), ``top_k``
        (default 50, 0 = off), ``top_p`` (default 1.0), then ``min_p``, ``typical_p``, ``epsilon_cutoff`` and ``eta_cutoff``
        (HF's MinP / Typical / Epsilon / Eta warpers in that order, each off by default; off too at min_p 0, typical_p
        >= 1 and a cutoff outside (0, 1), as in HF; min_p outside [0, 1] or typical_p <= 0 raises ValueError) — with a
        counter-based Philox stream keyed by ``seed`` (extension; default ``torch.initial_seed()``): the same seed
        reproduces the same tokens (csrc/sample.cu).  Every sampled mode below applies all of them.  Greedy, these
        keywords are ignored, as HF does.  ``top_h`` raises NotImplementedError.
        ``repetition_penalty``, ``no_repeat_ngram_size`` and ``min_new_tokens`` act as HF's logits processors, in that
        order and before the sampling warpers, on the last stage's GPU inside the decode graph (csrc/logits_process.cu).
        As in HF the history they look at is the whole ``input_ids`` row, pad tokens included, plus the generated tokens.
        ``input_ids`` [B,S] int64 on the first stage; returns [B,S+new] on every rank.
        An FP8 model (``quantization_config``, or an FP8 checkpoint) generates through every mode here with the tokens
        of the bf16 model over HF's dequantized weights: decode and verify steps of few rows stream the FP8 weights
        (``shard.fp8_gemv_rows``), larger ones dequantize each Linear before the bf16 GEMM.
        ``streamer``: object with ``put(tensor)`` / ``end()`` (HF BaseStreamer protocol), called on rank 0
        with each new token column, all batch rows (the reference streams row 0 only, worker.py:134-139).
        ``attention_mask``: a left-padded batch (HF's layout for batched generation) runs as ONE batch: columns that are
        pad in every row are dropped, and each row's pad slots are masked out of attention with its RoPE positions
        starting at its first real token.  The result keeps HF's layout [pads | prompt | new tokens | pad_token_id...].
        With ``do_sample`` a padded batch draws one stream per micro-batch slot, exactly as an unpadded batch does, so
        a row's tokens depend on the seed and its place in the batch, not on its prompt length.
        ``prompt_lookup_num_tokens=K`` (1..15; ``max_matching_ngram_size`` n, default 2): HF's prompt-lookup decoding for
        one row on one stage.  Each step drafts up to K tokens that followed an earlier occurrence of the last
        n-gram and verifies them with the current token as K+1 rows in one pass over the weights (csrc/prompt_lookup.cu);
        greedy, the output is greedy decoding's.  With ``do_sample`` every row draws a token from the model's warped
        distribution, and the drafts those draws agree with are kept with the draw that follows them, as in HF.
        ``self.timers["prompt_lookup_steps"]`` counts the verify steps.
        ``assistant_model=draft`` (another ``DistributedModel`` on this device, one stage; wrap an HF module as
        ``DistributedModel(hf_model, training=False)``), ``num_assistant_tokens=K`` (1..15): HF's assisted decoding for
        one row on one stage.  Each step the assistant drafts K tokens and the model verifies them with its current
        token as K+1 rows in one pass over its weights, keeping the agreeing prefix and its own next token, all on the
        GPU; greedy, the output is greedy decoding's.  With ``do_sample`` the assistant samples each draft from its own
        distribution warped by the same ``temperature`` / ``top_k`` / ``top_p``, and the model keeps it by speculative
        sampling (Leviathan et al.; csrc/sample.cu ``tl_spec_accept``).  Sampled with either draft source, every emitted
        token follows the model's warped distribution, as plain sampling's does, and a seed reproduces its tokens; they
        are other draws than plain sampling's for that seed (the streams: ml/stage.py STREAM_PL_ROWS).  The two models may differ in
        every dimension, the vocabulary included: an id one of them cannot embed reads its embedding row 0, which can
        only cost acceptance; sampled, an id outside the assistant's vocabulary has q = 0 and a draft outside the model's
        has p = 0 (rejected), which extends HF's rule, defined for equal vocabularies only.  Matching tokenizers are the
        caller's responsibility, as in HF.  Without ``num_assistant_tokens`` K is ASSISTED_DEFAULT_K, the K with the
        most expected tokens per ms on an H100 for a Qwen2.5-7B model and a Qwen2.5-0.5B assistant ASSUMING an
        agreement of 0.8 per draft token (not measured on real checkpoints); it changes speed only: never the greedy output,
        nor the distribution of the sampled one.
        ``num_assistant_tokens_schedule`` may only be "constant" and ``assistant_confidence_threshold`` only None.
        ``self.timers["assisted_steps"]`` counts the verify steps.
        ``return_dict_in_generate=True`` returns HF's ``GenerateDecoderOnlyOutput`` (transformers is imported then only):
        ``sequences`` is the tensor above; ``scores`` / ``logits`` (with ``output_scores`` / ``output_logits``, else None)
        are tuples of fp32 [B, V] tensors on the stage's device, one per generated column.  ``logits[c][r]`` is
        float(bf16 logit) of row r, the values that picked its token; ``scores[c][r]`` is HF's processed and warped row:
        greedy, the logits after the logits processors (-inf for a banned id); sampled, x / temperature (IEEE fp32
        division) on the sampler's kept set and -inf elsewhere, so the emitted token's score is always finite.  The last
        stage's picking kernels log them inside the decode graph (no added launch) into buffers that cost
        B * max_new_tokens * V * 4 bytes per kind (2.5 GB for 32 rows x 128 tokens x 152,064 ids); the returned tensors
        are copies, broadcast from the last rank, and cut where the EOS check cuts ``sequences``.  ``attentions``,
        ``hidden_states`` and ``past_key_values`` are None (HF returns its cache as ``past_key_values``).  After a row's
        EOS its entries are this model's continuation of its own tokens, where HF feeds ``pad_token_id``.
        Without ``return_dict_in_generate=True``, ``output_scores`` / ``output_logits`` are ignored, as in HF, and the call
        runs exactly as without them.  With prompt lookup or an assistant, with the grouped left-padded path of a stage
        without ``supports_kv_start``, or on a non-CUDA stage, ``return_dict_in_generate=True`` raises
        NotImplementedError.  ``compute_transition_scores`` turns ``scores`` into per-token log-probabilities."""
        input_ids = kwargs.pop("input_ids", args[0] if args else None)
        req, input_ids = self._request(input_ids, kwargs)
        if req.groups is not None:
            return self._generate_left_padded(input_ids, req)
        result = (self._generate_lookup if req.draft is not None else self._generate_batch)(input_ids, req)
        if req.out is not None:
            result, logs = result
        if req.pad_cols is not None and req.pad_cols.shape[1]:       # the dropped pad columns return in the result
            result = torch.cat([req.pad_cols.to(result.device), result], dim=1)
        if req.out is None:
            return result
        from transformers.generation import GenerateDecoderOnlyOutput
        return GenerateDecoderOnlyOutput(sequences=result, **logs)

    def _request(self, input_ids, kwargs: dict):
        """``generate``'s keywords as one _Request, and ``input_ids`` as the run sees it (without the columns that are pad
        in every row).  Every rank parses its own keywords and checks every combination of modes, and of a mode and its
        stage, before any stage work; then one broadcast hands every rank what only the first one knows: the prompt's
        shape and padding, the logits processors' starting history and the sampling seed (``torch.initial_seed()``
        unless given)."""
        link, st = self.link, self.stage
        max_new = int(kwargs.pop("max_new_tokens", 20))
        streamer = kwargs.pop("streamer", None)
        use_graph = kwargs.pop("use_graph", True)
        profile = kwargs.pop("profile", False)       # CUDA events around every decode launch -> self.timers["decode_busy_s"]
        sampling = None
        temperature, top_k, top_p = kwargs.pop("temperature", None), kwargs.pop("top_k", None), kwargs.pop("top_p", None)
        warp = {k: kwargs.pop(k, None) for k in ("min_p", "typical_p", "epsilon_cutoff", "eta_cutoff")}
        seed = kwargs.pop("seed", None)
        if kwargs.pop("do_sample", False):
            sampling = {"temperature": 1.0 if temperature is None else float(temperature), "top_k": 50 if top_k is None else int(top_k),
                        "top_p": 1.0 if top_p is None else float(top_p), "seed": int(torch.initial_seed() if seed is None else seed)}
            if sampling["temperature"] <= 0 or not (0 < sampling["top_p"] <= 1) or sampling["top_k"] < 0:
                raise ValueError(f"invalid sampling parameters {sampling}")
            sampling.update(_warpers(**warp))
        eos_token_id, pad_token_id = kwargs.pop("eos_token_id", None), kwargs.pop("pad_token_id", None)
        procs = _logits_processors(kwargs.pop("repetition_penalty", None), kwargs.pop("no_repeat_ngram_size", None),
                                   kwargs.pop("min_new_tokens", None), eos_token_id)
        mask = kwargs.pop("attention_mask", None)
        lookup = kwargs.pop("prompt_lookup_num_tokens", None)
        ngram = kwargs.pop("max_matching_ngram_size", None) if lookup is not None else None
        assistant = kwargs.pop("assistant_model", None)
        n_assist = kwargs.pop("num_assistant_tokens", None) if assistant is not None else None
        out = _output_flags(kwargs.pop("return_dict_in_generate", None), kwargs.pop("output_scores", None),
                            kwargs.pop("output_logits", None))
        _check_unconsumed(kwargs, "DistributedModel.generate")
        if assistant is not None and lookup is not None:
            # (HF drafts by prompt lookup here and ignores the assistant without a word)
            raise NotImplementedError("assistant_model together with prompt_lookup_num_tokens: pick one draft source")
        if out is not None and (lookup is not None or assistant is not None):
            raise NotImplementedError("return_dict_in_generate=True with prompt_lookup_num_tokens / assistant_model")
        if out is not None:
            _stage_supports(st, "scores", "return_dict_in_generate=True")
        pad_cols = kv_start = groups = None
        if link.first and mask is not None:
            if tuple(mask.shape) != tuple(input_ids.shape):
                raise ValueError(f"attention_mask shape {tuple(mask.shape)} != input_ids shape {tuple(input_ids.shape)}")
            if _stage_supports(st, "kv_start"):
                p = _left_pad_starts(mask)
                if p is not None:
                    pad_cols, kv_start = input_ids[:, :p[0]].cpu(), p[1]
                    input_ids = input_ids[:, p[0]:]
            else:
                groups = _left_pad_groups(mask)
        shape = tuple(input_ids.shape) if input_ids is not None else (1, 0)
        draft = None
        if assistant is not None:
            draft = _assisted(self, assistant, n_assist, shape, max_new, sampling, procs)
        elif lookup is not None:
            draft = _prompt_lookup(lookup, ngram, shape, max_new, self.max_seq, sampling, procs, self.world, st, eos_token_id)
        else:
            if sampling is not None:
                _stage_supports(st, "sampling", "do_sample=True")
            if procs is not None:
                _stage_supports(st, "processors", "repetition_penalty / no_repeat_ngram_size / min_new_tokens")
        history = None
        if procs is not None and link.first:         # the starting history: every column, the dropped pad columns too
            history = input_ids.cpu() if pad_cols is None else torch.cat([pad_cols, input_ids.cpu()], dim=1)
        if self.world > 1:
            shape, pad_cols, kv_start, groups, history, sampling = link.broadcast_object(
                (shape, pad_cols, kv_start, groups, history, sampling) if link.first else None)
        if groups is not None:                       # the grouped runs generate each real length in a run of its own:
            if procs is not None:                    # each row's history would lack its pads
                raise NotImplementedError("repetition_penalty / no_repeat_ngram_size / min_new_tokens with a left-padded "
                                          "batch need a stage with per-row key starts (supports_kv_start)")
            if out is not None:                      # the rows come back in separate runs
                raise NotImplementedError("return_dict_in_generate=True with a left-padded batch needs a stage with "
                                          "per-row key starts (supports_kv_start)")
            if streamer is not None:                 # the rows finish in separate runs
                raise NotImplementedError("streamer with a padded batch (rows finish in separate runs)")
        pad_token_id = None if pad_token_id is None else int(pad_token_id)
        return _Request(max_new, shape, sampling, tuple(_eos_list(eos_token_id)), pad_token_id, procs, draft, out, streamer,
                        use_graph, profile, pad_cols, kv_start, groups, history), input_ids

    def compute_transition_scores(self, sequences: torch.Tensor, scores, normalize_logits: bool = False) -> torch.Tensor:
        """HF ``compute_transition_scores`` without beams: [B, len(scores)] = each emitted token's score at its column,
        log-softmax normalised over the vocabulary first with ``normalize_logits`` (per-token log-probabilities from
        ``generate(..., return_dict_in_generate=True, output_scores=True)``; with ``do_sample`` they are those of the
        warped distribution).  The generated columns are the last len(scores) of ``sequences``."""
        T = len(scores)
        stacked = torch.stack(scores).reshape(T, -1).transpose(0, 1)          # [B*V, T], HF's layout
        V = scores[0].shape[-1]
        if normalize_logits:
            stacked = torch.nn.functional.log_softmax(stacked.reshape(-1, V, T), dim=1).reshape(-1, T)
        rows = torch.arange(scores[0].shape[0], device=sequences.device).view(-1, 1) * V
        return stacked.gather(0, sequences[:, sequences.shape[-1] - T:] + rows)

    def _generate_batch(self, input_ids, req: _Request):
        """One run of the batch: prefill every micro-batch, then the decode loop.  With logits processors, the last
        stage starts every row's history with ``req.history`` [B, S'] (``input_ids`` plus any pad columns dropped
        before the run).  Returns as ``_finish``."""
        link, st, cfg = self.link, self.stage, self.cfg
        B, S = req.shape
        max_new, streamer, procs, out = req.max_new, req.streamer, req.procs, req.out
        if _stage_supports(st, "scores"):            # off unless asked: the plain run keeps its launches
            st.set_score_log(bool(out and out["scores"]), bool(out and out["logits"]), B, max_new)
        if _stage_supports(st, "sampling"):
            st.set_sampling(req.sampling)           # the last stage draws; greedy (None) restores the argmax path
            if req.sampling is not None and st.has_head:
                st.sample_ctr.zero_()               # a seed names ONE stream: the same call reproduces its tokens
        if _stage_supports(st, "processors"):
            st.set_logits_processors(None if procs is None else dict(procs, prompt_len=req.history.shape[1]),
                                     0 if procs is None else req.history.shape[1] + max_new)
        n_mb = min(self.n_pipelines, B)
        while B % n_mb:                      # the largest micro-batch count <= n_pipelines that divides the batch
            n_mb -= 1
        b = B // n_mb
        if b > st.max_batch or S + max_new > st.max_seq:
            raise ValueError(f"stage sized for micro-batch<={st.max_batch}, T<={st.max_seq}; got {b}, {S + max_new}")
        dev = self.device
        t0 = time.perf_counter()
        out_tokens = torch.zeros(B, max_new, dtype=torch.int64, device=dev) if link.first else None
        ids_rows = [input_ids[m * b:(m + 1) * b].to(dev) for m in range(n_mb)] if link.first else [None] * n_mb

        # ---- prefill every micro-batch through the pipeline; the last stage produces the first new token
        multi = self.world > 1
        ring = self._peer_ring(n_mb) if multi else None
        if multi and ring is None:
            for g in st.slots:                       # NCCL kernels share the SMs during decode: no persistent all-SM kernel
                g.allow_chain = False
        if procs is not None and st.has_head:
            for m in range(n_mb):
                st.fill_history(m, req.history[m * b:(m + 1) * b].to(dev))
        if ring is not None:
            if max_new > ring.max_new:
                raise ValueError(f"max_new_tokens {max_new} exceeds the token log of the peer ring ({ring.max_new})")
            ring.reset()
        for m in range(n_mb):
            if link.first:
                x = st.embed(ids_rows[m])
            else:
                x = torch.empty(b, S, cfg.hidden, dtype=torch.bfloat16, device=dev)
                link.recv_prev(x)
            if req.kv_start is None:
                x = st.prefill(x, 0, m)
            else:
                x = st.prefill(x, 0, m, kv_start=req.kv_start[m * b:(m + 1) * b])
            if not link.last:
                link.send_next(x.clone())
            elif ring is not None:                         # first token straight into the first stage's mailbox
                st.head_argmax(x[:, -1, :].contiguous(), ring.first_ids_in[m][:b], m)
                ring.signal_ids(m)
            else:
                st.head_argmax(x[:, -1, :].contiguous(), st.ids_dec[m][:b], m)
                if multi:
                    link.send_up(st.ids_dec[m][:b].clone(), 0)
        if ring is not None:
            return self._decode_ring(ring, input_ids, req, b, n_mb, t0)
        # ---- decode rounds: micro-batches rotate through the stages; hidden [b,H] hops down, ids hop back up.
        # Sends are asynchronous; a slot's buffer is waited on only right before the next step overwrites it.
        sent_x = [None] * n_mb
        sent_ids = [None] * n_mb
        prof_events = []
        if req.profile:
            span = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            span[0].record()
        n_cols = max_new

        def collect(m, step):
            """first stage: ids of micro-batch m for column ``step`` (sent by the last stage in the previous round)"""
            if multi:
                link.wait(sent_x[m])                       # x_dec[m] still feeding the previous hop?
                link.recv_up(st.ids_dec[m][:b], self.world - 1)
            out_tokens[m * b:(m + 1) * b, step] = st.ids_dec[m][:b]

        for step in range(max_new):
            collected = False
            if req.eos and step and step % EOS_CHECK_EVERY == 0:
                # Stop once every row has emitted EOS (HF semantics).  The first stage takes this column's ids of EVERY
                # micro-batch first, so that no send is left without its posted receive when the ranks meet in the
                # broadcast below (a collective queued behind an unmatched point-to-point op could wait forever).
                if link.first:
                    for m in range(n_mb):
                        collect(m, step)
                collected = True
                flag = torch.zeros(1, dtype=torch.int32, device=dev)
                if link.first and _all_rows_finished(out_tokens[:, :step + 1], req.eos):
                    flag.fill_(1)
                if multi:
                    link.flush()
                    if torch.device(dev).type == "cuda":
                        torch.cuda.synchronize(dev)
                    link.broadcast(flag, 0)
                if int(flag.item()):
                    n_cols = step + 1
                    if streamer is not None and link.first:
                        streamer.put(out_tokens[:, step].cpu())
                    break
            for m in range(n_mb):
                if link.first:
                    if not collected:
                        collect(m, step)
                    if streamer is not None and m == n_mb - 1:
                        streamer.put(out_tokens[:, step].cpu())         # all rows of this step, one column
                if step == max_new - 1:
                    continue
                if not link.first:
                    link.wait(sent_x[m])
                    link.recv_prev(st.x_dec[m][:b])
                if link.last and multi:
                    link.wait(sent_ids[m])
                if req.profile:
                    ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                    ev[0].record()
                st.decode(m, b, req.use_graph)
                if req.profile:
                    ev[1].record()
                    prof_events.append(ev)
                if not link.last:
                    sent_x[m] = link.send_next(st.x_dec[m][:b])
                elif multi:
                    sent_ids[m] = link.send_up(st.ids_dec[m][:b], 0)
        link.flush()
        if req.profile:
            span[1].record()
            torch.cuda.synchronize()
            self.timers["decode_span_s"] = span[0].elapsed_time(span[1]) * 1e-3
            self.timers["decode_busy_s"] = sum(a.elapsed_time(b_) for a, b_ in prof_events) * 1e-3
        return self._finish(req, input_ids, out_tokens, n_cols, t0)
