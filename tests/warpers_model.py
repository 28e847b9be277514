"""A float64 row model of the sampler's min_p / typical_p / epsilon / eta stages (csrc/sample.cu), HF's warper chain on
fp32 copies, and the draw model the device tests compare against (tests/rowwise_cases.py RowModel).

The model applies the kernels' documented rules exactly in float64: after top-k / top-p (rowwise_cases.sample_row_model)
each stage keeps one interval of values of the current set, with weights w = exp(x/T - x_ref) over that set (x_ref: the
set's top value / T, rebased after typical as the kernels do).  Every threshold carries an error band that covers the
device's fp32 / fixed-point rounding and HF's fp32 arithmetic; a row is pinned when no token lies inside any band, and
on a pinned row the device, the model and HF must keep the same tokens."""
import math
from dataclasses import dataclass

import numpy as np
import torch

from tests.rowwise_cases import ARG_REL, EXP_REL, RowModel, sample_row_model

REL = 2.0 ** -16            # relative band of every mass / weight comparison (fp32 softmax sums in HF, float weights here)
FAULTS = ("min_p_extra_bin", "typical_shift", "eps_before_min_p", "eta_whole_row", "kept_weight_no_hi")


@dataclass
class Warp:
    min_p: float = 0.0
    typical_p: float = 1.0
    epsilon: float = 0.0
    eta: float = 0.0

    def kwargs(self) -> dict:
        return dict(min_p=self.min_p, typical_p=self.typical_p, epsilon=self.epsilon, eta=self.eta)


def processed_values(row_bf16: torch.Tensor, present=None, banned=None, penalty=1.0) -> np.ndarray:
    """fp32 values as the kernels see them: the bf16 logit, then HF's repetition penalty and the bans"""
    x = row_bf16.float().numpy().astype(np.float32)
    if present is not None:
        pen = np.float32(penalty)
        x = np.where(present, np.where(x < 0, x * pen, x / pen).astype(np.float32), x)
    if banned is not None:
        x = np.where(banned, np.float32(-np.inf), x)
    return x


def warp_row(x: np.ndarray, temperature, kept0: np.ndarray, w: Warp, fault=None):
    """(kept mask, pinned, s_ref) after the four stages on the set kept0 (top-k / top-p's); x fp32 values"""
    it = np.float32(1.0) / np.float32(temperature)
    s = (x.astype(np.float32) * it).astype(np.float64)
    kept = kept0.copy()
    pinned = True
    fin = np.isfinite(s)

    def weights(k):
        ref = s[k & fin].max()
        with np.errstate(invalid="ignore", over="ignore"):
            return np.where(k & fin, np.exp(np.where(k & fin, s - ref, -np.inf)), 0.0), ref

    def cut(k, t, wt, Zb=None):
        """keep w >= t on the set k (w: the set's weights), plus the set's top value"""
        nonlocal pinned
        top = s[k & fin].max()
        keep = k & ((wt >= t) | (s == top))
        if np.any(k & (s != top) & (np.abs(wt - t) <= REL * max(t, 1e-300) + 1e-12 * (Zb or 1.0))):
            pinned = False
        return keep

    if w.min_p > 0:
        wt, _ = weights(kept)
        t = w.min_p * 1.0
        k2 = cut(kept, t, wt)
        if fault == "min_p_extra_bin":               # one distinct value below the boundary kept too
            below = np.unique(s[kept & ~k2 & fin])
            if len(below):
                k2 = k2 | (kept & (s == below[-1]))
        pre_min_p = kept
        kept = k2
    else:
        pre_min_p = kept
    if w.typical_p < 1:
        wt, ref = weights(kept)
        Z = wt.sum()
        a = np.where(kept & fin, s - ref, 0.0)
        mean = (wt * a).sum() / Z
        d = np.where(kept, np.abs(mean - a), np.inf)
        d = np.where(kept & ~fin, np.inf, d)
        order = np.argsort(d, kind="stable")
        ds, ws = d[order], wt[order]
        uniq, first = np.unique(ds, return_index=True)
        gmass = np.add.reduceat(ws, first)
        closer = np.concatenate([[0.0], np.cumsum(gmass)[:-1]])
        lim = w.typical_p * Z
        keep_g = closer < lim
        gi = int(np.nonzero(keep_g)[0][-1])
        if fault == "typical_shift":
            gi = min(gi + 1, len(uniq) - 1)
        dstar = uniq[gi]
        tol_d = 2.0 ** -19 * (1.0 + abs(mean) + np.abs(a[kept & fin]).max())
        near = kept & fin & (np.abs(d - dstar) <= tol_d) & (d != dstar)
        if np.any(near) or np.any(np.abs(closer - lim) <= REL * Z):
            pinned = False
        kept = kept & (d <= dstar)

    def mass_on(k, ref):
        with np.errstate(invalid="ignore", over="ignore"):
            return float(np.where(k & fin, np.exp(np.where(k & fin, s - ref, -np.inf)), 0.0).sum())

    if w.epsilon > 0:
        wt, ref = weights(kept)
        Z = mass_on(pre_min_p if fault == "eps_before_min_p" else kept, ref)
        kept = cut(kept, w.epsilon * Z, wt, Z)
    if w.eta > 0:
        base = np.ones_like(kept) if fault == "eta_whole_row" else kept
        wb, refb = weights(base)
        Zb = wb.sum()
        ab = np.where(base & fin, s - refb, 0.0)
        H = math.log(Zb) - float((wb * ab).sum()) / Zb
        eps = min(w.eta, math.sqrt(w.eta) * math.exp(-H))
        wt, _ = weights(kept)
        Z = wt.sum()
        kept = cut(kept, eps * Z, wt, Z)
    return kept, pinned, s


def warped_model(row_bf16: torch.Tensor, temperature, top_k, top_p, w: Warp, proc=False, present=None, banned=None,
                 penalty=1.0, fault=None) -> RowModel:
    """rowwise_cases.sample_row_model's top-k / top-p, then the four stages: the kept interval and the draw's weights
    relative to the kept top (fixed point 2^40 on the processed path), as the kernels weigh them"""
    base = sample_row_model(row_bf16, temperature, top_k, top_p, proc=proc, present=present, banned=banned, penalty=penalty)
    if base.banned_all:
        return base
    x = processed_values(row_bf16, present, banned, penalty) if proc else row_bf16.float().numpy().astype(np.float32)
    kept, pinned, s = warp_row(x, temperature, base.kept, w, fault)
    ref = s[kept].max()
    arg = np.where(kept, s - ref, 0.0)
    wt = np.where(kept, np.exp(arg), 0.0)
    rel = EXP_REL + ARG_REL * (2 * np.abs(arg) + np.abs(s))
    rel = np.where(np.isfinite(rel), rel, 0.0)
    if proc:
        wt = np.floor(wt * 2.0 ** 40)
        err = np.where(kept, wt * rel + 1.0, 0.0)
    else:
        wt = np.where(wt < 2.0 ** -126, 0.0, wt)
        err = np.where(kept, wt * rel + 2.0 ** -126, 0.0)
    C = np.cumsum(wt)
    return RowModel(kept, wt, err, C, float(C[-1]), proc, pinned and base.pinned)


def hf_warped(scores_fp32: torch.Tensor, temperature, top_k, top_p, w: Warp) -> torch.Tensor:
    """HF's sampling warpers (transformers' _get_logits_processor order, min_tokens_to_keep 1) on [N, V] fp32 scores
    that already went through the logits processors; returns the warped scores"""
    from transformers.generation import logits_process as L
    chain = []
    if temperature != 1.0:
        chain.append(L.TemperatureLogitsWarper(temperature))
    if top_k:
        chain.append(L.TopKLogitsWarper(top_k))
    if top_p < 1.0:
        chain.append(L.TopPLogitsWarper(top_p))
    if w.min_p > 0:
        chain.append(L.MinPLogitsWarper(w.min_p))
    if w.typical_p < 1.0:
        chain.append(L.TypicalLogitsWarper(w.typical_p))
    if 0.0 < w.epsilon < 1.0:
        chain.append(L.EpsilonLogitsWarper(w.epsilon))
    if 0.0 < w.eta < 1.0:
        chain.append(L.EtaLogitsWarper(w.eta))
    ids = torch.zeros(scores_fp32.shape[0], 1, dtype=torch.long)
    out = scores_fp32.float().clone()
    for p in chain:
        out = p(ids, out)
    return out


def replay_kept_weight(rm: RowModel, s: np.ndarray, fault=None) -> np.ndarray:
    """tl_spec_accept's kept_weight over a row from the model: exp(s - ref) inside [lo, hi], else 0; with the fault
    ``kept_weight_no_hi`` every value >= lo counts, as if hi_key were ignored"""
    ks = s[rm.kept]
    lo, hi = ks.min(), ks.max()
    inside = (s >= lo) if fault == "kept_weight_no_hi" else ((s >= lo) & (s <= hi))
    with np.errstate(over="ignore", invalid="ignore"):
        return np.where(inside & np.isfinite(s), np.exp(np.where(inside, s - hi, 0.0)), 0.0)
