"""Model-level parity of the CUDA shard executor against the CPU oracle (same seeded weights and tokens).

Tolerance for multi-op chains (a whole layer, the whole model): a bf16 pipeline is chaotic at the ulp level — a
1e-4 input perturbation flips the rounding of a few percent of the elements of every later op — so the reference's
OWN bf16 output sits 5e-3..8e-3 (rel-L2) from exact fp32 math after ONE layer on these weights, and its two
attention paths (eager / sdpa, identical GEMMs) differ by 3e-3..6e-3 (measured, tools/diag.py).  The 1e-3 figure of
the north star is therefore applied per op (tests/test_kernels_gpu.py); for chains the criteria are
  (i)  accuracy: rel-L2(gpu, fp32 oracle) <= 1.25 x rel-L2(bf16 oracle, fp32 oracle)  — the CUDA path is no
       further from exact math than the reference's CPU bf16 path is;
  (ii) agreement: rel-L2(gpu, bf16 oracle) <= 2 x rel-L2(bf16 oracle, fp32 oracle)  — two independent bf16
       evaluations of the same function (expected sqrt(2) x).
Token ids: exact wherever the oracle's
top-2 logit margin exceeds MARGIN (random-init logits are nearly flat; a margin below the bf16 noise of the logits
cannot be resolved by ANY bf16 implementation, including the reference on another CPU).
"""
import pytest
import torch
import torch.nn.functional as F

from oracle import shard_oracle as O
from tensorlink_b200.ml import configs as C
from tensorlink_b200.ml.weights import init_state_dict, synthetic_tokens

pytestmark = pytest.mark.gpu
CASES = [C.TINY_QWEN2, C.TINY_QWEN2_D128, C.TINY_QWEN3]
MARGIN = 0.05


def make(cfg, **kw):
    from tensorlink_b200.ml import DistributedModel
    kw.setdefault("max_seq", 256)
    return DistributedModel(cfg, training=False, **kw)


def _fp32_state(sd):
    return {k: v.float() for k, v in sd.items()}


def _chain_check(tag, got, ref_bf16, ref_f32):
    e_ref, e_gpu, mutual = O.rel_l2(ref_bf16, ref_f32), O.rel_l2(got, ref_f32), O.rel_l2(got, ref_bf16)
    print(f"{tag}: gpu-vs-fp32 {e_gpu:.3e}  oracle_bf16-vs-fp32 {e_ref:.3e}  gpu-vs-oracle_bf16 {mutual:.3e}")
    assert e_gpu <= 1.25 * e_ref, "criterion (i) accuracy"
    assert mutual <= 2.0 * e_ref, "criterion (ii) agreement"


@pytest.mark.parametrize("cfg", CASES, ids=lambda c: c.name)
def test_forward_logits_vs_oracle(cfg):
    sd = init_state_dict(cfg)
    ids = synthetic_tokens(cfg, 2, 40)
    with torch.no_grad():
        ref = O.OracleModel(cfg, sd, "sdpa_math").logits(ids)
        ref32 = O.OracleModel(cfg, _fp32_state(sd), "sdpa_math").logits(ids)     # same bf16-rounded weights, fp32 math
    got = make(cfg)(ids).logits.cpu()
    _chain_check(f"{cfg.name} logits", got, ref, ref32)
    safe = (lambda t: (t[..., 0] - t[..., 1]) > MARGIN)(ref32.topk(2, -1).values)
    assert torch.equal(got.float().argmax(-1)[safe], ref32.argmax(-1)[safe])


@pytest.mark.parametrize("cfg", CASES, ids=lambda c: c.name)
def test_per_layer_teacher_forced(cfg):
    from tensorlink_b200.ml.shard import CudaLayerGroup, ShardParams
    sd = init_state_dict(cfg)
    ids = synthetic_tokens(cfg, 2, 33)
    m = O.OracleModel(cfg, sd, "sdpa_math")
    m32 = O.OracleModel(cfg, _fp32_state(sd), "sdpa_math")
    B, S = ids.shape
    per_layer = []
    with torch.no_grad():
        m.hidden(ids, per_layer=per_layer)
        x0 = F.embedding(ids, m.embed)
        cos, sin = O.rope_tables(cfg, torch.arange(S)[None].expand(B, -1), torch.float32)
    inputs = [x0] + per_layer[:-1]
    for li in range(cfg.n_layers):
        with torch.no_grad():   # exact math on the SAME (bf16) layer input
            y32 = O.decoder_layer(cfg, m32.layers[li], inputs[li].float(), cos, sin, "sdpa_math")
        p = ShardParams(cfg, [li], False, False, "cuda")
        p.load_hf_state_dict(sd)
        grp = CudaLayerGroup(cfg, p, 2, 64)
        out = grp(hidden_states=inputs[li].cuda(), past_len=0)
        assert set(out) == {"hidden_states", "past_len"}           # kwargs ∪ outputs (injector.py:252-260)
        _chain_check(f"{cfg.name} layer {li}", out["hidden_states"].cpu(), per_layer[li], y32)


def _check_ids(got, ref, margins, prompt_len):
    """exact up to the first step whose oracle margin is below MARGIN; a mismatch before that is a failure."""
    new_got, new_ref = got[:, prompt_len:], ref[:, prompt_len:]
    n_exact = 0
    for b in range(ref.shape[0]):
        for s in range(new_ref.shape[1]):
            if margins[b, s] < MARGIN:
                break                      # beyond an unresolvable step the sequences may legitimately fork
            assert new_got[b, s] == new_ref[b, s], f"row {b} step {s}: margin {margins[b, s]:.3f}"
            n_exact += 1
    return n_exact


@pytest.mark.parametrize("cfg", CASES, ids=lambda c: c.name)
@pytest.mark.parametrize("B", [1, 2])
def test_generate_greedy_ids(cfg, B):
    sd = init_state_dict(cfg)
    ids = synthetic_tokens(cfg, B, 12)
    ref, margins = O.OracleModel(cfg, sd, "sdpa_math").generate(ids, 24, return_margins=True)
    dm = make(cfg, max_batch=B)
    got = dm.generate(ids, max_new_tokens=24).cpu()
    got_nograph = dm.generate(ids, max_new_tokens=24, use_graph=False).cpu()
    assert got.shape == ref.shape and torch.equal(got[:, :12], ids)
    assert torch.equal(got, got_nograph)                      # CUDA-graph replay == eager launches, bit for bit
    n = _check_ids(got, ref, margins, 12)
    print(f"{cfg.name} B={B}: {n} of {B * 24} steps verified exact (margin >= {MARGIN}); "
          f"full-sequence match: {torch.equal(got, ref)}")
    assert n >= 1


@pytest.mark.parametrize("cfg", [C.TINY_QWEN2_D128], ids=lambda c: c.name)
def test_generate_teacher_forced_exact(cfg):
    """Feed the ORACLE's generated sequence back as a prompt: every position's greedy choice must agree wherever the
    oracle margin allows, independent of earlier forks."""
    sd = init_state_dict(cfg)
    ids = synthetic_tokens(cfg, 2, 8)
    ref, margins = O.OracleModel(cfg, sd, "sdpa_math").generate(ids, 40, return_margins=True)
    logits = make(cfg)(ref[:, :-1]).logits.cpu().float()
    pred = logits.argmax(-1)[:, 7:]                            # predictions for the 40 generated positions
    safe = margins >= MARGIN
    assert safe.float().mean() > 0.3
    assert torch.equal(pred[safe], ref[:, 8:][safe])


def test_batched_decode_gemm_path():
    """B = 16 rows decode through the wgmma GEMM path; rows are independent, so row i must equal a B=1 run."""
    cfg = C.TINY_QWEN2_D128
    ids = synthetic_tokens(cfg, 16, 10)
    big = make(cfg, max_batch=16).generate(ids, max_new_tokens=12).cpu()
    sd = init_state_dict(cfg)
    ref, margins = O.OracleModel(cfg, sd, "sdpa_math").generate(ids, 12, return_margins=True)
    assert _check_ids(big, ref, margins, 10) >= 16


def test_micro_batched_generate_equals_single():
    cfg = C.TINY_QWEN2
    ids = synthetic_tokens(cfg, 4, 9)
    a = make(cfg, max_batch=4).generate(ids, max_new_tokens=10).cpu()
    b = make(cfg, max_batch=4, n_pipelines=2).generate(ids, max_new_tokens=10).cpu()
    sd = init_state_dict(cfg)
    ref, margins = O.OracleModel(cfg, sd, "sdpa_math").generate(ids, 10, return_margins=True)
    assert _check_ids(a, ref, margins, 9) >= 4 and _check_ids(b, ref, margins, 9) >= 4


def test_full_size_qwen25_05b_properties():
    """BASELINE config 2 at full size (the oracle would take minutes): size-independent properties.
    (1) graph replay == eager launches; (2) incremental decode == one-shot prefill (KV-cache consistency):
    the ids produced step by step must be the argmax of a single forward over the final sequence wherever the
    one-shot top-2 margin is resolvable; (3) generation is deterministic run to run."""
    cfg = C.QWEN25_05B
    dm = make(cfg, max_batch=1, max_seq=128, init="device")
    ids = synthetic_tokens(cfg, 1, 32)
    a = dm.generate(ids, max_new_tokens=24).cpu()
    b = dm.generate(ids, max_new_tokens=24, use_graph=False).cpu()
    c = dm.generate(ids, max_new_tokens=24).cpu()
    assert torch.equal(a, b) and torch.equal(a, c)
    logits = dm(a[:, :-1]).logits.cpu().float()
    top2 = logits.topk(2, -1).values
    safe = ((top2[..., 0] - top2[..., 1]) > MARGIN)[:, 31:]
    assert torch.equal(logits.argmax(-1)[:, 31:][safe], a[:, 32:][safe])
    assert safe.float().mean() > 0.2


@pytest.mark.parametrize("max_seq", [2048, 4096])
def test_long_context_decode_consistency(max_seq):
    """BASELINE configs 3 / 5 context lengths (seq 2048 / 4096) on the full-size 0.5B model: a long prompt, then
    incremental decode through the fused (T_max <= 2048) or the split-KV (T_max = 4096) attention path must pick the
    argmax of ONE forward over the final sequence wherever that forward's top-2 margin is resolvable, and the graph
    replay must equal eager launches."""
    cfg = C.QWEN25_05B
    S, new = max_seq - 40, 24
    dm = make(cfg, max_batch=1, max_seq=max_seq, init="device")
    ids = synthetic_tokens(cfg, 1, S)
    a = dm.generate(ids, max_new_tokens=new).cpu()
    b = dm.generate(ids, max_new_tokens=new, use_graph=False).cpu()
    assert torch.equal(a, b)
    logits = dm(a[:, :-1]).logits[:, S - 1:].cpu().float()
    top2 = logits.topk(2, -1).values
    safe = (top2[..., 0] - top2[..., 1]) > MARGIN
    assert safe.float().mean() > 0.2
    assert torch.equal(logits.argmax(-1)[safe], a[:, S:][safe])


def test_batch32_decode_rows_independent():
    """BASELINE config 5 batch (32 rows per step, wgmma GEMM + split-K decode path) at full 0.5B width: every row
    of the batched generation equals the same prompt generated alone (B = 1, GEMV path) wherever the one-shot top-2
    margin is resolvable."""
    cfg = C.QWEN25_05B
    ids = synthetic_tokens(cfg, 32, 48)
    big = make(cfg, max_batch=32, max_seq=128, init="device")
    out = big.generate(ids, max_new_tokens=16).cpu()
    logits = big(out[:, :-1]).logits[:, 47:].cpu().float()
    top2 = logits.topk(2, -1).values
    safe = (top2[..., 0] - top2[..., 1]) > MARGIN
    assert safe.float().mean() > 0.2
    assert torch.equal(logits.argmax(-1)[safe], out[:, 48:][safe])
    one = make(cfg, max_batch=1, max_seq=128, init="device")
    for r in (0, 13, 31):
        alone = one.generate(ids[r:r + 1], max_new_tokens=16).cpu()
        # rows agree until the first step whose margin is below the threshold (after that the contexts differ)
        ok = safe[r].clone()
        first_unsafe = int((~ok).nonzero()[0]) if (~ok).any() else 16
        assert torch.equal(alone[0, 48:48 + first_unsafe], out[r, 48:48 + first_unsafe]), r
