"""Parity at BASELINE scale: the CUDA path against the CPU oracle on full-size shapes, and directly against the golden
vectors the reference's own ``LayerGroupModule`` produced.

  (a) full-size Qwen2.5-0.5B (BASELINE config 2): logits of a 32-token prompt and greedy ids, same seeded weights;
  (b) one decoder layer at Qwen2.5-7B width and one at Qwen3-8B width + the full-vocabulary lm_head: a 192-token
      prefill (wgmma GEMMs, wgmma attention), then 4 single-token decode steps through the
      weight-streaming GEMV path with the fused (T_max <= 2048) and the split-KV (T_max = 4096) decode attention;
  (c) the CUDA shard operator teacher-forced on ``tests/golden/ref_layergroup_*.pt`` hop by hop.

Criteria are the chain criteria of tests/test_model_gpu.py (a bf16 pipeline is compared with the reference's OWN bf16
distance from exact fp32 math, measured in the same test): accuracy <= 1.25x, agreement <= 2x; greedy ids exact
wherever the fp32 oracle's top-2 margin exceeds MARGIN.
"""
import glob
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import shard_oracle as O
from tensorlink_b200.ml import configs as C
from tensorlink_b200.ml.weights import init_state_dict, synthetic_tokens

pytestmark = pytest.mark.gpu
MARGIN = 0.05
GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "ref_layergroup_*_sdpa.pt")))


def _f32(sd):
    return {k: v.float() for k, v in sd.items()}


def _chain(tag, got, ref16, ref32, acc=1.25, agree=2.0):
    e_ref, e_gpu, mutual = O.rel_l2(ref16, ref32), O.rel_l2(got, ref32), O.rel_l2(got, ref16)
    print(f"{tag}: gpu-vs-fp32 {e_gpu:.3e}  oracle_bf16-vs-fp32 {e_ref:.3e}  gpu-vs-oracle_bf16 {mutual:.3e}")
    assert e_gpu <= acc * e_ref, f"{tag}: accuracy"
    assert mutual <= agree * e_ref, f"{tag}: agreement"


def _ids_exact_where_resolvable(got, ref, margins, prompt):
    n = 0
    for b in range(ref.shape[0]):
        for s in range(ref.shape[1] - prompt):
            if margins[b, s] < MARGIN:
                break
            assert got[b, prompt + s] == ref[b, prompt + s], f"row {b} step {s} margin {margins[b, s]:.3f}"
            n += 1
    return n


# ---------------------------------------------------------------------------------------------- (a) config 2, full size
def test_full_size_qwen25_05b_vs_oracle():
    from tensorlink_b200.ml import DistributedModel
    cfg = C.QWEN25_05B
    sd = init_state_dict(cfg)
    ids = synthetic_tokens(cfg, 1, 32)
    m16, m32 = O.OracleModel(cfg, sd, "sdpa_math"), O.OracleModel(cfg, _f32(sd), "sdpa_math")
    with torch.no_grad():
        ref16, ref32 = m16.logits(ids), m32.logits(ids)
    dm = DistributedModel(cfg, training=False, max_batch=1, max_seq=128)         # init="seeded": the oracle's weights
    got = dm(ids).logits.cpu()
    _chain("Qwen2.5-0.5B logits [1,32,V]", got, ref16, ref32)
    top2 = ref32.topk(2, -1).values
    safe = (top2[..., 0] - top2[..., 1]) > MARGIN
    assert torch.equal(got.float().argmax(-1)[safe], ref32.argmax(-1)[safe])
    new = 24
    ref_ids, margins = m32.generate(ids, new, return_margins=True)
    out = dm.generate(ids, max_new_tokens=new).cpu()
    n = _ids_exact_where_resolvable(out, ref_ids, margins, 32)
    print(f"Qwen2.5-0.5B greedy ids: {n} of {new} steps verified exact against the fp32 oracle (margin >= {MARGIN}); "
          f"full match: {torch.equal(out, ref_ids)}")
    assert n >= 1


# ---------------------------------------------------------------------------------------------- (b) 7B / 8B width layer
def _one_layer_case(base):
    cfg = base.scaled(name=base.name + "-1layer", n_layers=1)
    sd = init_state_dict(cfg)
    return cfg, sd


@pytest.mark.parametrize("base", [C.QWEN25_7B, C.QWEN3_8B], ids=lambda c: c.name)
@pytest.mark.parametrize("max_seq", [512, 4096], ids=["fused-decode-attn", "splitkv-decode-attn"])
def test_full_width_layer_and_head_vs_oracle(base, max_seq):
    """embed -> one full-width decoder layer -> final norm -> lm_head (V = 152k): prefill of S tokens, then 4 decode
    steps teacher-forced with the ORACLE's tokens, so every step compares the same function on both sides."""
    from tensorlink_b200.ml import DistributedModel
    cfg, sd = _one_layer_case(base)
    S, steps = 192, 4
    ids = synthetic_tokens(cfg, 1, S)
    m16, m32 = O.OracleModel(cfg, sd, "sdpa_math"), O.OracleModel(cfg, _f32(sd), "sdpa_math")
    dm = DistributedModel(cfg, training=False, max_batch=1, max_seq=max_seq)
    st = dm.stage
    with torch.no_grad():
        c16, c32 = O.KVCache(), O.KVCache()
        h16, h32 = m16.hidden(ids, cache=c16), m32.hidden(ids, cache=c32)
        tail = slice(S - 8, S)
        l16 = F.linear(O.rmsnorm(h16[:, tail], m16.norm, cfg.rms_eps), m16.head)
        l32 = F.linear(O.rmsnorm(h32[:, tail], m32.norm, cfg.rms_eps), m32.head)
    # ---- prefill through the product path (wgmma GEMMs + wgmma attention), logits through head_logits
    x = st.prefill(st.embed(ids.cuda()), 0, 0)
    _chain(f"{cfg.name} layer output [1,{S},H]", x.cpu(), h16, h32)
    got = st.head_logits(x[0, tail].contiguous()).cpu()[None]
    _chain(f"{cfg.name} logits (last 8 positions)", got, l16, l32)
    # ---- decode steps (GEMV path + decode attention), teacher-forced on the fp32 oracle's greedy tokens
    nxt = l32[:, -1].argmax(-1)
    for s in range(steps):
        with torch.no_grad():
            d16 = m16.logits(nxt[:, None], cache=c16, past_len=S + s)[:, -1]
            d32 = m32.logits(nxt[:, None], cache=c32, past_len=S + s)[:, -1]
        st.ids_dec[0][:1].copy_(nxt.cuda())
        st.decode(0, 1, use_graph=(s % 2 == 0))                 # graph replay and eager launches both
        got = st.logits_dec[:1].cpu()
        _chain(f"{cfg.name} decode step {s} logits", got, d16, d32)
        top2 = d32.float().topk(2, -1).values
        if float(top2[0, 0] - top2[0, 1]) > MARGIN:
            assert int(st.ids_dec[0][0]) == int(d32.argmax(-1)[0])
        nxt = d32.argmax(-1)


# ---------------------------------------------------------------------------------------------- (c) golden vectors
@pytest.mark.parametrize("path", GOLDEN, ids=os.path.basename)
def test_cuda_shards_vs_reference_layergroup_golden(path):
    """The CUDA shard operator on the inputs the reference's ``LayerGroupModule`` saw (embedding of the golden ids for
    the first shard, the reference's own hop for every later one), compared with the hop the reference produced.
    Tolerance: the spread between the reference's own eager and sdpa runs of the same shard."""
    from tensorlink_b200.ml.shard import CudaLayerGroup, ShardParams
    from tensorlink_b200.ml.stage import CudaStage
    g = torch.load(path)
    ge = torch.load(path.replace("_sdpa.pt", "_eager.pt"))
    cfg = C.get_config(g["cfg"])
    sd = init_state_dict(cfg, seed=g["seed"])
    ids = g["input_ids"]
    B, S = ids.shape
    x_in = F.embedding(ids, sd["model.embed_tokens.weight"])
    for (a, b), ref, ref_e in zip(g["bounds"], g["hops"], ge["hops"]):
        p = ShardParams(cfg, list(range(a, b)), False, False, "cuda")
        p.load_hf_state_dict(sd)
        grp = CudaLayerGroup(cfg, p, B, 64)
        out = grp(hidden_states=x_in.cuda(), past_len=0)["hidden_states"].cpu()
        floor = O.rel_l2(ref_e, ref)
        err = O.rel_l2(out, ref)
        print(f"{os.path.basename(path)} layers {a}..{b - 1}: gpu-vs-reference {err:.3e}  reference eager-vs-sdpa {floor:.3e}")
        assert err <= 1.5 * floor + 1e-6
        x_in = ref                                           # teacher-forced on the reference's own hop
    head = CudaStage(cfg, [], False, True, "cuda", B, 64, state_dict=sd)
    logits = head.head_logits(g["hops"][-1].cuda().reshape(B * S, cfg.hidden)).view(B, S, cfg.vocab)[:, -4:].cpu()
    assert O.rel_l2(logits, g["logits"]) <= 1e-3            # one Linear on identical inputs: per-op tolerance
    assert torch.equal(logits.float().argmax(-1), g["logits"].float().argmax(-1))


# ---------------------------------------------------------------------------------------------- (d) training at full width
def _oracle_grads(cfg, sd0, ids, dtype):
    sd = {k: v.to(dtype).clone().requires_grad_(True) for k, v in sd0.items()}
    if cfg.tied:
        sd["lm_head.weight"] = sd["model.embed_tokens.weight"]
    loss, _ = O.OracleModel(cfg, sd, "sdpa_math").loss(ids, ids)
    loss.backward()
    return float(loss.detach()), {k: v.grad for k, v in sd.items() if v.grad is not None}


@pytest.mark.parametrize("base", [C.QWEN25_7B, C.QWEN3_8B], ids=lambda c: c.name)
@pytest.mark.parametrize("n_mb", [1, 2], ids=["fused-head", "split-head-deferred-w"])
def test_full_width_training_step_vs_oracle_autograd(base, n_mb):
    """One optimizer step's worth of gradients through a full-width decoder layer and the 152k-row lm_head (wgmma
    GEMMs with MN-major operands at the real K / N, attention backward at 28/4 and 32/8 heads of 128, fused CE over the
    real vocabulary) against the oracle's autograd in fp32; the oracle's own bf16 run sets the yardstick.  n_mb = 2 runs
    the pipelined form: deferred weight gradients and the split head backward (ml/train.py)."""
    from tensorlink_b200.ml import DistributedModel
    cfg, sd = _one_layer_case(base)
    ids = synthetic_tokens(cfg, 2, 64)
    loss32, g32 = _oracle_grads(cfg, sd, ids, torch.float32)
    loss16, g16 = _oracle_grads(cfg, sd, ids, torch.bfloat16)
    dm = DistributedModel(cfg, training=True, n_pipelines=n_mb, max_batch=2, max_seq=64, optimizer=torch.optim.Adam)
    opt = dm.create_optimizer(lr=1e-4)
    opt.zero_grad()
    out = dm(ids, labels=ids)
    out.loss.backward()
    torch.cuda.synchronize()
    assert dm.stage.trainer.head_split == (n_mb > 1)
    print(f"{cfg.name} n_mb={n_mb}: loss gpu {float(out.loss.detach()):.6f} oracle_bf16 {loss16:.6f} oracle_fp32 {loss32:.6f}")
    assert abs(float(out.loss.detach()) - loss32) <= max(2 * abs(loss16 - loss32), 2e-3)
    got = dm.stage.params.hf_state_dict(grads=True)
    for name, ref in g32.items():
        e_ref, e_gpu = O.rel_l2(g16[name], ref), O.rel_l2(got[name].cpu(), ref)
        print(f"  {name}: gpu-vs-fp32 {e_gpu:.3e} oracle_bf16-vs-fp32 {e_ref:.3e}")
        assert e_gpu <= 1.5 * e_ref + 2e-3, name
