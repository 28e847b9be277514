"""One pipeline stage on one H100: parameters + per-micro-batch shard operators + captured decode graphs.

This is the worker half of the reference's hot path (/root/reference/tensorlink/ml/worker.py):
``load_module`` (:452-505) -> ``CudaStage.__init__``; ``_handle_forward`` (:297-357) -> ``prefill`` / ``decode``;
``_handle_generate`` (:359-441) -> the decode graph.  There is no polling loop and no IPC: the stage is driven
in-process by ``DistributedModel`` and neighbours are reached through ``StageLink``.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch

from .. import native as nat
from .configs import ShardModelConfig
from .shard import CudaLayerGroup, ShardParams, gemv_max_rows

# Philox streams of one sampled generate call, all keyed by its ``seed``: stream s draws with the key seed + GOLDEN * s
# (mod 2^64).  The plain head sampler of slot m is stream m (so the first token of a drafted run is slot 0's); the
# drafted verify steps take the streams below, which no slot index reaches.  GOLDEN is odd, so distinct streams have
# distinct keys.  Within a stream a (Philox row, counter) pair is used once:
#   STREAM_PL_ROWS   prompt lookup: row i of the K+1 verify rows draws on Philox row i, counter pl["ctr"][i]
#   STREAM_DRAFTS    the assistant's drafts: Philox row 0, counter pl["ctr"][16], one step per draft
#   STREAM_ACCEPT    tl_spec_accept: u_i on Philox row i, the final draw on row 16, counter pl["ctr"][17], one step a round
GOLDEN = 0x9E3779B97F4A7C15
STREAM_PL_ROWS, STREAM_DRAFTS, STREAM_ACCEPT = 2 ** 32 - 1, 2 ** 32 - 2, 2 ** 32 - 3
CTR_DRAFTS, CTR_ACCEPT = nat.VERIFY_MAX_ROWS, nat.VERIFY_MAX_ROWS + 1


def stream_seed(seed: int, stream: int) -> int:
    return (seed + GOLDEN * stream) & (2 ** 64 - 1)


# the sampling dict's optional warpers (generate's min_p / typical_p / epsilon_cutoff / eta_cutoff) as the keyword
# arguments of nat.sample / sample_proc / spec_accept; a dict carries only the active ones
WARPER_KEYS = ("min_p", "typical_p", "epsilon", "eta")


def warpers(sampling: dict) -> dict:
    return {k: sampling[k] for k in WARPER_KEYS if k in sampling}


class CudaStage:
    def __init__(self, cfg: ShardModelConfig, layer_ids, has_embed: bool, has_head: bool, device,
                 max_batch: int, max_seq: int, n_slots: int = 1, training: bool = False,
                 state_dict: Optional[Dict[str, torch.Tensor]] = None, seed: int = 1234, init: str = "seeded",
                 max_tokens: Optional[int] = None, quantization: Optional[dict] = None):
        """``quantization``: ml/fp8.parse_quantization_config's result for an FP8 model (weight-only FP8 decoder
        Linears), None for bf16."""
        nat.require_device()
        self.cfg = cfg
        self.device = torch.device(device)
        self.has_embed, self.has_head = has_embed, has_head
        self.supports_training, self.trainer = bool(training), None
        self.supports_kv_start = True       # prefill(kv_start=...): left-padded batches run as one batch
        self.params = ShardParams(cfg, layer_ids, has_embed, has_head, self.device, with_grad=training,
                                  fp8=quantization is not None)
        if state_dict is not None:
            self.params.load_hf_state_dict(state_dict)
        elif init == "device":
            self.params.init_on_device(seed)
        else:
            self.params.init_seeded(seed)
        self.max_batch, self.max_seq = max_batch, max_seq
        self.slots: List[CudaLayerGroup] = [CudaLayerGroup(cfg, self.params, max_batch, max_seq, max_tokens)
                                            for _ in range(n_slots)]
        dev = self.device
        # decode-time fixed buffers (graph inputs/outputs), one set per slot
        self.x_dec = [torch.zeros(max_batch, cfg.hidden, dtype=torch.bfloat16, device=dev) for _ in range(n_slots)]
        self.ids_dec = [torch.zeros(max_batch, dtype=torch.int64, device=dev) for _ in range(n_slots)]
        self.graphs: Dict[tuple, torch.cuda.CUDAGraph] = {}
        if has_head:
            self.head_ws = torch.empty(max(nat.lmhead_ws(min(max_batch, 8), cfg.vocab), max_batch * 64 * 8 + 256),
                                       dtype=torch.uint8, device=dev)
            self.logits_dec = torch.empty(max_batch, cfg.vocab, dtype=torch.bfloat16, device=dev)
            self.hn = torch.empty(max_batch, cfg.hidden, dtype=torch.bfloat16, device=dev)
            self.head_ctr = nat.gemv_counters(device=dev)        # the decode lm_head GEMV's ticket counter
            self.sampling: Optional[dict] = None        # set by generate(do_sample=True): temperature / top_k / top_p / seed
                                                        # (+ the active WARPER_KEYS)
            self.sample_ctr = torch.zeros(n_slots, max_batch, dtype=torch.int32, device=dev)
            self.sample_ws: Optional[torch.Tensor] = None
            # logits processors (set_logits_processors): per slot and row a token history on the device -- log
            # [n_slots, max_batch, L], length, presence bitmap of V bits -- and the parameters (penalty, n, ...)
            self.procs: Optional[dict] = None
            self.lp_flags = 0
            self.hist_log: Optional[torch.Tensor] = None
            self.hist_len = self.hist_bits = self.lp_params = self.lp_ws = None
            # prompt-lookup decoding (prompt_lookup_begin): the verify step's buffers, allocated on first use; the draft
            # source is the history's n-grams, or an assistant stage (assisted decoding)
            self.pl: Optional[dict] = None
            self.pl_K = 0
            self.pl_assistant: Optional["CudaStage"] = None
            # as an assistant (assist_draft): its 2-row catch-up input and hidden rows, allocated on first use
            self.asst: Optional[dict] = None
            # generate's output_scores / output_logits (set_score_log): fp32 logs [columns, rows, V] of the scores and the
            # raw logits, and per slot the log column {column, exit word} the picking kernel writes and advances
            self.score_log: Optional[dict] = None
            self.log_mode: Tuple[bool, bool] = (False, False)

    # ------------------------------------------------------------------------------------------ pieces
    def embed(self, ids: torch.Tensor) -> torch.Tensor:
        """[B,S] int64 -> [B,S,H]  (host-side ``embed_tokens`` in the reference, module.py:1023-1056)."""
        return nat.embed_fwd(ids.contiguous(), self.params.v["embed"])

    def prefill(self, hidden: torch.Tensor, past_len: int = 0, slot: int = 0, kv_start=None) -> torch.Tensor:
        """``kv_start``: per-row leading pad slots of a left-padded batch (CudaLayerGroup.prefill)."""
        return self.slots[slot].prefill(hidden, past_len, kv_start)

    def head_logits(self, hidden: torch.Tensor) -> torch.Tensor:
        """final norm + lm_head over [N,H] -> bf16 logits [N,V]."""
        return self._lm_head(hidden.contiguous())

    def _lm_head(self, hidden: torch.Tensor, logits: Optional[torch.Tensor] = None, hn: Optional[torch.Tensor] = None,
                 counter: Optional[torch.Tensor] = None) -> torch.Tensor:
        """final norm + lm_head of [n,H] rows into ``logits`` [n,V] (a new tensor when None): up to gemv_max_rows() rows
        the GEMV with the norm fused (``counter``: its ticket block), above that the norm into ``hn`` [n,H], then the GEMM."""
        cfg, v = self.cfg, self.params.v
        if hidden.shape[0] <= gemv_max_rows():
            return nat.gemv(hidden, v["head"], out=logits, norm_w=v["norm"], eps=cfg.rms_eps, counter=counter)
        return nat.gemm(nat.rmsnorm_fwd(hidden, v["norm"], cfg.rms_eps, out=hn), v["head"], out=logits)

    def _pick(self, hidden: torch.Tensor, ids_out: torch.Tensor, logits: torch.Tensor, hn: torch.Tensor,
              head_ws: torch.Tensor, sample: Optional[tuple] = None, hist: Optional[tuple] = None, log=None):
        """final norm + lm_head of [n,H] rows into ``logits`` (``_lm_head``), then one token per row into ``ids_out``:
        the argmax, or with ``sample`` = (sampling dict, counters, sampler workspace, Philox key) a draw from the warped
        row.  ``hist`` = (log, length, bits, params) of the rows' token histories: both act on HF's processed scores
        and append the picked id.  ``log``: a score log (``_log``).  Greedy without either, up to gemv_max_rows() rows, is
        the fused tl_lmhead_argmax (the decode hot path); the others run the GEMV and the picking kernel as two calls."""
        cfg, v = self.cfg, self.params.v
        if sample is None and hist is None and log is None and hidden.shape[0] <= gemv_max_rows():
            nat.lmhead_argmax(hidden, v["head"], v["norm"], cfg.rms_eps, ids_out, logits, head_ws, self.head_ctr)
            return
        self._lm_head(hidden, logits, hn, self.head_ctr)
        if sample is None and hist is None:
            nat.argmax_bf16(logits, ids_out, head_ws, log=log)
        elif sample is None:
            nat.argmax_proc(logits, ids_out, *hist, self.lp_ws, self.lp_flags, score_log=log)
        else:
            s, ctr, ws, key = sample
            warp = (s["temperature"], s["top_k"], s["top_p"])
            if hist is None:
                nat.sample(logits, ids_out, ctr, ws, *warp, key, log=log, **warpers(s))
            else:
                nat.sample_proc(logits, ids_out, *hist, ctr, self.lp_ws, *warp, key, self.lp_flags, score_log=log,
                                **warpers(s))

    def set_sampling(self, sampling: Optional[dict]):
        """None = greedy.  Changing the mode drops the captured decode graphs (the launch sequence differs)."""
        if not self.has_head or sampling == self.sampling:
            return
        self.sampling = sampling
        self.graphs.clear()
        self.sample_ctr.zero_()
        if sampling is not None and self.sample_ws is None:
            self.sample_ws = torch.empty(nat.sample_ws(self.max_batch), dtype=torch.uint8, device=self.device)

    def set_logits_processors(self, procs: Optional[dict], length: int = 0):
        """HF's repetition penalty / no-repeat n-gram / min-new-tokens on the last stage; None = off.  ``procs``: penalty,
        ngram, min_new, eos (ids), prompt_len (history entries that are prompt); ``length``: the longest history of the
        run (prompt width + max_new_tokens).  Switching on or off, or the ban set on or off, drops the captured decode
        graphs (the launch sequence differs); the values live in device memory, so changing them keeps the graphs."""
        if not self.has_head:
            return
        flags = 0 if procs is None else (nat.LP_BAN if procs["ngram"] > 0 or (procs["min_new"] > 0 and procs["eos"]) else 0)
        if (procs is None) != (self.procs is None) or flags != self.lp_flags:
            self.graphs.clear()
        self.procs, self.lp_flags = procs, flags
        if procs is None:
            return
        dev, V = self.device, self.cfg.vocab
        if self.lp_ws is None:
            self.lp_ws = torch.empty(nat.logits_proc_ws(self.max_batch, V), dtype=torch.uint8, device=dev)
            self.lp_params = torch.zeros(nat.LP_PARAMS, dtype=torch.int32, device=dev)
        self._ensure_history(length)
        self.lp_params.copy_(nat.lp_params(procs["penalty"], procs["ngram"], procs["min_new"], procs["prompt_len"],
                                           procs["eos"] if procs["min_new"] > 0 else []))

    def _ensure_history(self, length: int):
        """The token history of every slot and row, holding at least ``length`` tokens (the logits processors' and
        prompt lookup's)."""
        n_slots, dev, V = len(self.slots), self.device, self.cfg.vocab
        if self.hist_len is None:
            self.hist_len = torch.zeros(n_slots, self.max_batch, dtype=torch.int32, device=dev)
            self.hist_bits = torch.zeros(n_slots, self.max_batch, (V + 31) // 32, dtype=torch.int32, device=dev)
        if self.hist_log is None or self.hist_log.shape[2] < length:
            self.hist_log = torch.zeros(n_slots, self.max_batch, max(length, self.max_seq), dtype=torch.int32, device=dev)
            self.graphs.clear()                      # the captured kernels hold the old log's address

    def set_score_log(self, scores: bool, logits: bool, rows: int = 0, n_cols: int = 0):
        """Log every picked row's scores (HF's processed and warped values) and / or raw logits (fp32 of the bf16 logits)
        into fp32 buffers [n_cols, rows, V]: the head of slot m writes its rows at m * (its batch) in the column its
        counter names, and advances it.  Both False = off.  The buffers only grow; growing them or changing the mode
        drops the captured decode graphs (they hold the buffer addresses and the launch's kernels).  Zeroes the columns."""
        if not self.has_head:
            return
        mode = (bool(scores), bool(logits))
        if mode != self.log_mode:
            self.graphs.clear()
        self.log_mode = mode
        if not any(mode):
            return
        dev, V = self.device, self.cfg.vocab
        lg = self.score_log
        if lg is None:
            lg = self.score_log = {"col": torch.zeros(len(self.slots), 2, dtype=torch.int32, device=dev),
                                   "scores": None, "logits": None}
        shape = (max(n_cols, 1), max(rows, 1))
        for kind, on in zip(("scores", "logits"), mode):
            t = lg[kind]
            if on and (t is None or t.shape[0] < shape[0] or t.shape[1] < shape[1]):
                old = (0, 0) if t is None else t.shape[:2]
                lg[kind] = None                      # free the old buffer first
                lg[kind] = torch.empty(max(shape[0], old[0]), max(shape[1], old[1]), V, dtype=torch.float32, device=dev)
                self.graphs.clear()
        lg["col"].zero_()

    def _log(self, slot: int, B: int):
        """slot's score log as the native picking calls take it, or None when off."""
        if not any(self.log_mode):
            return None
        lg = self.score_log
        return (lg["logits"] if self.log_mode[1] else None, lg["scores"] if self.log_mode[0] else None, lg["col"][slot],
                slot * B)

    def score_log_copy(self, kind: str, rows: int, n_cols: int) -> torch.Tensor:
        """Columns 0..n_cols-1 of rows 0..rows-1 of the ``kind`` ("scores" / "logits") log: a new fp32 tensor
        [n_cols, rows, V] (the next run does not change it)."""
        return self.score_log[kind][:n_cols, :rows].clone()

    def fill_history(self, slot: int, prompt: torch.Tensor):
        """Row r of ``slot`` starts its token history with ``prompt[r]`` (int64 [b, S] on this device, pad columns included)."""
        nat.history_fill(prompt.contiguous(), self.hist_log[slot], self.hist_len[slot], self.hist_bits[slot], self.cfg.vocab)

    def head_argmax(self, hidden: torch.Tensor, ids_out: torch.Tensor, slot: int = 0):
        """next token for [B,H] rows -> ids_out [B] int64: greedy (bit-exact target: torch.argmax of bf16 logits) or, after
        ``set_sampling``, one draw per row from the warped distribution (csrc/sample.cu).  With logits processors on, both
        act on HF's processed scores and append the picked id to the row's history."""
        B, s = hidden.shape[0], self.sampling
        sample = None if s is None else (s, self.sample_ctr[slot], self.sample_ws, stream_seed(s["seed"], slot))
        hist = None if self.procs is None else (self.hist_log[slot], self.hist_len[slot], self.hist_bits[slot], self.lp_params)
        self._pick(hidden, ids_out, self.logits_dec[:B], self.hn[:B], self.head_ws, sample, hist, self._log(slot, B))

    # ------------------------------------------------------------------------------------------ decode step
    def _decode_body_ring(self, slot: int, B: int, ring):
        """The decode step of a multi-stage pipeline with the hops on peer memory (p2p/peer.py): wait for this slot's
        input in the local mailbox, run the layers, let the last kernel store into the neighbour's mailbox, signal."""
        grp = self.slots[slot]
        if self.has_embed:
            ring.wait_ids(slot, bump=grp.kvlen_dev)              # the opening wait also counts the new key in
            ring.log_token(slot, B)
            x = self.x_dec[slot][:B]
            nat.embed_fwd(ring.ids_in[slot][:B], self.params.v["embed"], out=x)
        else:
            ring.wait_x(slot, bump=grp.kvlen_dev)
            x = ring.x_in[slot][:B]
        if self.has_head:
            grp.decode_step_inplace(x, advance=False)
            self.head_argmax(x, ring.first_ids_in[slot][:B], slot)
            ring.signal_ids(slot, bump=grp.pos_dev)              # the closing signal also advances the cache position
        else:
            grp.decode_step_inplace(x, out=ring.next_x_in[slot][:B], advance=False)
            ring.signal_x(slot, bump=grp.pos_dev)

    def _decode_body(self, slot: int, B: int, ring=None):
        if ring is not None:
            self._decode_body_ring(slot, B, ring)
            return
        x = self.x_dec[slot][:B]
        if self.has_embed:
            nat.embed_fwd(self.ids_dec[slot][:B], self.params.v["embed"], out=x)
        self.slots[slot].decode_step_inplace(x)
        if self.has_head:
            self.head_argmax(x, self.ids_dec[slot][:B], slot)

    def decode(self, slot: int, B: int, use_graph: bool = True, ring=None):
        """One token for slot's rows: [embed ->] layers [-> norm + lm_head + argmax], as ONE graph launch.
        Inputs/outputs are the fixed buffers ``ids_dec[slot]`` / ``x_dec[slot]``, or the mailboxes of ``ring``."""
        if not use_graph:
            self._decode_body(slot, B, ring)
            return
        ragged = self.slots[slot].ragged          # the captured launches differ (the _rows kernels, no decode chain)
        key = (slot, B, ragged, self.log_mode if self.has_head else None) + (() if ring is None else (id(ring),))
        # (the warm-up runs without the ring: it must never touch the mailboxes)
        self._replay(key, lambda: self._decode_body(slot, B, ring), lambda: self._decode_body(slot, B), slot)

    def _step_state(self, slot: int) -> List[torch.Tensor]:
        """Every piece of device state a decode or verify step of ``slot`` moves: cache position and length, the step's
        ids / hidden buffers, the sampler counters, the token histories, the score-log columns, the verify step's
        counters and the assistant's position and length.  A graph's warm-up restores all of them (restoring one the
        step does not touch is harmless; a missed one would corrupt the first replay)."""
        grp = self.slots[slot]
        state = [grp.pos_dev, grp.kvlen_dev, self.ids_dec[slot], self.x_dec[slot]]
        if not self.has_head:
            return state
        state.append(self.sample_ctr)
        if self.hist_len is not None:
            state += [self.hist_len, self.hist_bits]
        if self.score_log is not None:
            state.append(self.score_log["col"])
        if self.pl is not None:
            state += [self.pl[k] for k in ("count", "in_ids", "n_cand", "ctr") if k in self.pl]
        if self.pl_assistant is not None:
            state += [self.pl_assistant.slots[0].pos_dev, self.pl_assistant.slots[0].kvlen_dev]
        return state

    def _replay(self, key, body, warm_up, slot: int):
        """Replay the graph of ``key``, capturing ``body`` first if there is none: ``warm_up`` runs once outside capture
        (first-use attribute setting, tensor-map caches), then every tensor of ``_step_state(slot)`` gets its value
        back, so the warm-up consumes no draw, joins no history and logs no column.  Capture does not execute."""
        g = self.graphs.get(key)
        if g is None:
            state = self._step_state(slot)
            saved = [t.clone() for t in state]
            side = torch.cuda.Stream(device=self.device)
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                warm_up()
            torch.cuda.current_stream().wait_stream(side)
            for t, s in zip(state, saved):
                t.copy_(s)
            torch.cuda.synchronize(self.device)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                body()
            self.graphs[key] = g
        g.replay()

    # ------------------------------------------------------------------------------------------ prompt-lookup decoding
    def _whole_model(self) -> bool:
        return self.has_embed and self.has_head and len(self.slots[0].layer_ids) == self.cfg.n_layers

    def prompt_lookup_begin(self, seq: torch.Tensor, K: int, ngram: int, max_length: int, eos=(),
                            assistant: Optional["CudaStage"] = None):
        """Start a prompt-lookup run of slot 0, row 0 right after its prefill: ``seq`` (int64 [1, S+1] on this device) is
        the prompt and the first generated token, whose key is not cached yet (pos_dev = S).  The row's history becomes
        ``seq`` and the output log starts with the first token (count 1).  Each verify step then drafts K tokens from
        the history (largest n-gram ``ngram``, EOS ids ``eos``) and runs K+1 rows; the history never grows past
        ``max_length`` (prompt + max_new_tokens).
        ``assistant``: assisted decoding instead.  That stage (another model on this device, its slot 0 prefilled with
        the prompt) drafts K tokens greedily in every step (``assist_draft``); ``ngram`` and ``eos`` are unused.
        After ``set_sampling`` the steps sample: prompt lookup draws every verify row from its warped distribution and
        keeps the drafts the draws agree with (HF's sampled candidate check); an assistant samples its drafts and the
        step keeps them by speculative sampling (``tl_spec_accept``).  The streams are described at STREAM_PL_ROWS;
        their counters restart at 0 here."""
        if not self._whole_model() or (assistant is not None and not assistant._whole_model()):
            raise NotImplementedError("prompt lookup decoding runs on a stage that holds the whole model")
        if assistant is self:
            raise ValueError("a stage cannot be its own assistant (the two would share one KV cache)")
        if assistant is not None and assistant.device != self.device:
            raise NotImplementedError(f"an assistant on {assistant.device} for a stage on {self.device}")
        if not 1 <= K <= nat.PL_MAX_DRAFT:
            raise ValueError(f"prompt lookup drafts 1..{nat.PL_MAX_DRAFT} tokens per step, got {K}")
        # a captured assisted step holds its assistant's buffer addresses (its cache key holds the stage itself, so the
        # addresses stay valid): keep the graphs of one assistant only
        for key in [k for k in self.graphs if k[0] == "assist" and k[2] is not assistant]:
            del self.graphs[key]
        self.pl_assistant = assistant
        if assistant is not None:
            eos = ()                                 # an accepted EOS draft is cut on the host, as a decoded one
        dev, H, V, R = self.device, self.cfg.hidden, self.cfg.vocab, nat.VERIFY_MAX_ROWS
        if self.pl is None:
            self.pl = {"in_ids": torch.zeros(R, dtype=torch.int64, device=dev),       # last token + drafts (+ filler)
                       "ids": torch.zeros(R, dtype=torch.int64, device=dev),          # the model's token after each row
                       "n_cand": torch.zeros(1, dtype=torch.int32, device=dev),
                       "count": torch.zeros(1, dtype=torch.int32, device=dev),        # tokens in the output log
                       "params": torch.zeros(nat.PL_PARAMS, dtype=torch.int32, device=dev),
                       "x": torch.zeros(R, H, dtype=torch.bfloat16, device=dev),
                       "hn": torch.zeros(R, H, dtype=torch.bfloat16, device=dev),
                       "logits": torch.zeros(R, V, dtype=torch.bfloat16, device=dev),
                       "head_ws": torch.empty(max(nat.lmhead_ws(8, V), R * 64 * 8 + 256), dtype=torch.uint8, device=dev),
                       "out_log": torch.zeros(0, dtype=torch.int64, device=dev)}
        pl = self.pl
        if self.sampling is not None and "ctr" not in pl:
            pl["ctr"] = torch.zeros(R + 2, dtype=torch.int32, device=dev)        # see STREAM_PL_ROWS
            pl["sample_ws"] = torch.empty(nat.sample_ws(R), dtype=torch.uint8, device=dev)
            pl["spec_ws"] = torch.empty(nat.spec_accept_ws(nat.PL_MAX_DRAFT), dtype=torch.uint8, device=dev)
        if "ctr" in pl:
            pl["ctr"].zero_()
        S = seq.shape[1] - 1
        if pl["out_log"].numel() < max_length - S:
            pl["out_log"] = torch.zeros(max(max_length - S, 64), dtype=torch.int64, device=dev)
            self.graphs.clear()                      # the captured accept kernel holds the old log's address
        self._ensure_history(max_length)
        self.fill_history(0, seq.contiguous())
        pl["params"].copy_(nat.pl_params(ngram, max_length, eos))
        pl["out_log"][:1].copy_(seq[0, -1:])
        pl["count"].fill_(1)
        self.pl_K = int(K)

    def _verify_body(self, draft: bool = True):
        """draft (n-gram kernel, or the assistant's K tokens) -> embed K+1 ids -> layers -> final norm + lm_head + argmax
        of every row -> accept.  Sampled (``set_sampling``): the lm_head writes the K+1 logits rows, then one draw per row
        (prompt lookup) or speculative sampling against the assistant's rows, then the same accept."""
        pl, grp, cfg, v = self.pl, self.slots[0], self.cfg, self.params.v
        K = self.pl_K
        n = K + 1
        s, asst = self.sampling, self.pl_assistant
        log, length, bits = self.hist_log[0, 0], self.hist_len[0, :1], self.hist_bits[0, 0]
        if draft and asst is not None:
            asst.assist_draft(log, length, pl["in_ids"], K, None if s is None else (s, pl["ctr"][CTR_DRAFTS:CTR_DRAFTS + 1]))
            pl["n_cand"].fill_(K)
        elif draft:
            nat.pl_draft(log, length, pl["params"], K, pl["in_ids"], pl["n_cand"])
        x, ids, logits = pl["x"][:n], pl["ids"][:n], pl["logits"][:n]
        nat.embed_fwd(pl["in_ids"][:n], v["embed"], out=x)
        grp.verify_step_inplace(x)
        if s is not None and asst is not None:
            self._lm_head(x, logits, pl["hn"][:n], self.head_ctr)
            nat.spec_accept(logits, asst.asst["q"][:K], pl["in_ids"], pl["n_cand"], pl["ctr"][CTR_ACCEPT:CTR_ACCEPT + 1],
                            ids, pl["spec_ws"], s["temperature"], s["top_k"], s["top_p"], stream_seed(s["seed"], STREAM_ACCEPT),
                            **warpers(s))
        else:
            sample = None if s is None else (s, pl["ctr"][:n], pl["sample_ws"], stream_seed(s["seed"], STREAM_PL_ROWS))
            self._pick(x, ids, logits, pl["hn"][:n], pl["head_ws"], sample)
        nat.pl_accept(ids, pl["in_ids"], pl["n_cand"], log, length, bits, cfg.vocab, pl["params"], pl["out_log"], pl["count"],
                      grp.pos_dev, grp.kvlen_dev, K)

    def prompt_lookup_step(self, use_graph: bool = True):
        """One verify step (``prompt_lookup_begin``), as ONE graph launch per K: it emits 1..K+1 tokens into the output
        log, or none once the history holds max_length tokens."""
        if not use_graph:
            self._verify_body()
            return
        asst, sampled = self.pl_assistant, self.sampling is not None
        key = ("verify", self.pl_K + 1, sampled) if asst is None else ("assist", self.pl_K + 1, asst, sampled)
        self._replay(key, self._verify_body, self._verify_body, 0)

    def prompt_lookup_count(self) -> int:
        """Tokens in the output log (synchronises with the device)."""
        return int(self.pl["count"].item())

    def prompt_lookup_tokens(self, start: int, end: int) -> torch.Tensor:
        """Output-log entries start..end-1 (int64, on the host)."""
        return self.pl["out_log"][start:end].cpu()

    def verify_drafts(self, drafts) -> List[int]:
        """One eager verify step with the caller's drafts (at most K) in place of the history's: in_ids = [last history
        token, *drafts, filler].  Returns the tokens it emitted: the accepted drafts and the model's next token."""
        pl = self.pl
        K = self.pl_K
        if len(drafts) > K:
            raise ValueError(f"{len(drafts)} drafts for a verify step of K={K}")
        nat.pl_draft(self.hist_log[0, 0], self.hist_len[0, :1], pl["params"], K, pl["in_ids"], pl["n_cand"])
        if drafts:
            pl["in_ids"][1:1 + len(drafts)].copy_(torch.as_tensor(list(drafts), dtype=torch.int64))
        pl["n_cand"].fill_(len(drafts))
        c0 = self.prompt_lookup_count()
        self._verify_body(draft=False)
        return self.prompt_lookup_tokens(c0, self.prompt_lookup_count()).tolist()

    def verify_round(self) -> Tuple[List[int], List[int]]:
        """One eager verify step with the run's own draft source (n-grams or the assistant).  Returns its drafts and
        the tokens it emitted.  A sampled step leaves what its draws read: the counters ``pl["ctr"]``, the target's rows
        ``pl["logits"][:K+1]`` and the assistant's rows ``asst["q"][:K]``."""
        c0 = self.prompt_lookup_count()
        self._verify_body()
        drafts = self.pl["in_ids"][1:1 + int(self.pl["n_cand"].item())].tolist()
        return drafts, self.prompt_lookup_tokens(c0, self.prompt_lookup_count()).tolist()

    # ------------------------------------------------------------------------------------------ assisted decoding
    def assist_draft(self, log: torch.Tensor, length: torch.Tensor, in_ids: torch.Tensor, K: int,
                     sample: Optional[tuple] = None):
        """This stage as the assistant of another model's verify step (``prompt_lookup_begin(assistant=self)``): emit into
        the current stream, graph-capturable, the greedy drafts in_ids[1..K] after the target's history (``log`` int32
        [L], ``length`` int32 [1], on the target).  With P = length - 1, slot 0's cache must hold the history's keys up
        to slot P-2 (the prompt's prefill, then earlier rounds).  The round rewrites slots P-1 and P from the history's
        last two tokens as one 2-row verify step, whose last row gives in_ids[1], then feeds in_ids[i] at slot P+i for
        i = 1..K-1 as decode steps, each giving in_ids[i+1].  Slots above P that hold rejected drafts are overwritten
        by later rounds before they are read.
        ``sample`` = (sampling dict, counter int32[1]): draft i is drawn instead from this model's warped row (the
        target's temperature / top_k / top_p, stream STREAM_DRAFTS), which stays in ``asst["q"][i]`` for the target's
        speculative sampling."""
        grp, v, dev = self.slots[0], self.params.v, self.device
        if self.asst is None:
            self.asst = {"in": torch.zeros(2, dtype=torch.int64, device=dev),
                         "x": torch.zeros(2, self.cfg.hidden, dtype=torch.bfloat16, device=dev)}
        a = self.asst
        if sample is not None and "q" not in a:
            a["q"] = torch.zeros(nat.PL_MAX_DRAFT, self.cfg.vocab, dtype=torch.bfloat16, device=dev)
            a["ws"] = torch.empty(nat.sample_ws(1), dtype=torch.uint8, device=dev)

        def head(h, out, i):
            if sample is None:
                self._pick(h, out, self.logits_dec[:1], self.hn[:1], self.head_ws)
            else:
                s, ctr = sample
                self._pick(h, out, a["q"][i:i + 1], self.hn[:1], self.head_ws,
                           (s, ctr, a["ws"], stream_seed(s["seed"], STREAM_DRAFTS)))

        nat.assist_prep(log, length, a["in"], in_ids, grp.pos_dev, grp.kvlen_dev)      # pos = kv_len = P-1
        nat.embed_fwd(a["in"], v["embed"], out=a["x"])
        grp.verify_step_inplace(a["x"])
        head(a["x"][1:], in_ids[1:2], 0)
        nat.advance_pos(grp.pos_dev, grp.kvlen_dev, 2)                                  # pos = kv_len = P+1
        x = self.x_dec[0][:1]
        for i in range(1, K):
            nat.embed_fwd(in_ids[i:i + 1], v["embed"], out=x)
            grp.decode_step_inplace(x)
            head(x, in_ids[i + 1:i + 2], i)

    def check(self):
        for g in self.slots:
            g.check()

    def n_decode_launches(self, B: int, ring: bool = False) -> int:
        """Kernel launches inside one decode step of this stage (for bench.py's gpu_launches claim)."""
        fused = self.slots[0].T_max <= self.slots[0].FUSED_DECODE_MAX_T
        gemv = B <= self.slots[0].gemv_rows()
        if self.slots[0].chain_ok(B):
            n = self.slots[0].n_chain_launches() + 2       # qkv of the first layer + one persistent launch per layer group
        elif self.slots[0].dq_ok(B):
            # first qkv + per layer: attention (1 fused / 3), o, gate/up, [down + next qkv] as one chain launch
            n = 1 + len(self.slots[0].layer_ids) * (3 + (1 if fused else 3)) + 2
        else:
            # GEMV path: 4 Linears + attention (1 fused / 3); batched: 4 GEMMs + 3 split-K reduce(+norm) passes + attention
            n = len(self.slots[0].layer_ids) * ((7 if gemv else 10) - (2 if fused else 0)) + 2 + (0 if gemv else 1)
            if self.params.fp8:      # a second FP8 GEMV pass above 4 rows; the GEMM path dequantizes each Linear first
                n += len(self.slots[0].layer_ids) * 4 * ((B > 4) if gemv else 1)
        if ring:
            n += (3 if self.has_embed else 2) - 2    # wait (+ token log) + signal, which also do the two position updates
        if self.has_embed:
            n += 1
        if self.has_head:
            n += 3 if B <= gemv_max_rows() else 4
        return n
