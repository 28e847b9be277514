"""Training on padded batches: ``dm(ids, attention_mask=mask, labels=labels).loss.backward()``.

The step is compared with fp32 autograd of the masked oracle (tests/padded_oracle.py) under the criteria of
tests/test_train_gpu.py::test_training_step_vs_oracle_autograd.  S = 48 runs the mma.sync attention backward, S = 700
the wgmma one over 11 query tiles.  Pad tokens must not matter at all: their ids, the gradient they receive and the
way the mask reaches the loss are checked bit for bit."""
import pytest
import torch

from oracle import shard_oracle as O
from tensorlink_b200.ml import configs as C
from tensorlink_b200.ml.weights import init_state_dict, synthetic_tokens
from tests.padded_oracle import MaskedOracleModel, mask_shift_labels

pytestmark = pytest.mark.gpu
CFGS = [C.TINY_QWEN2, C.TINY_QWEN2_D128, C.TINY_QWEN3]


def padded(cfg, B, S, kind, pad_id=None, seed=0):
    """(ids, mask, labels) with HF collator labels (-100 on pad positions).  kind: left / right / mixed (left, right,
    both sides and unpadded rows).  Real lengths spread over [S/8, S]."""
    ids = synthetic_tokens(cfg, B, S, seed=seed)
    mask = torch.zeros(B, S, dtype=torch.int64)
    for r in range(B):
        L = max(1, S - ((r + 1) * 7 * S) // (8 * B))
        k = kind if kind != "mixed" else ("left", "right", "both", "none")[r % 4]
        a = {"left": S - L, "right": 0, "both": (S - L) // 2, "none": 0}[k]
        mask[r, a:a + (S if k == "none" else L)] = 1
    if pad_id is None:
        pad_id = min(set(range(cfg.vocab)) - set(ids[mask == 1].tolist()))      # occurs only as padding
    ids = ids.masked_fill(mask == 0, pad_id)
    return ids, mask, ids.masked_fill(mask == 0, -100)


def _dm(cfg, n_mb, B, S, seed=1234):
    from tensorlink_b200.ml import DistributedModel
    dm = DistributedModel(cfg, training=True, n_pipelines=n_mb, max_batch=B, max_seq=max(64, S), optimizer=torch.optim.Adam,
                          seed=seed)
    return dm, dm.create_optimizer(lr=1e-3)


def _step(dm, opt, ids, mask, labels):
    """forward, backward and one Adam step: (loss, gradient arena, parameter arena)"""
    opt.zero_grad()
    out = dm(ids, attention_mask=mask, labels=labels) if mask is not None else dm(ids, labels=labels)
    out.loss.backward()
    p = dm.stage.params
    p.grad_settle()
    grad = p.grad.clone()
    opt.step()
    if hasattr(opt, "wait"):
        opt.wait()
    torch.cuda.synchronize()
    return float(out.loss), grad, p.flat.clone()


def _oracle_grads(cfg, ids, mask, labels, dtype):
    sd = {k: v.to(dtype).clone().requires_grad_(True) for k, v in init_state_dict(cfg).items()}
    if cfg.tied:
        sd["lm_head.weight"] = sd["model.embed_tokens.weight"]
    loss, _ = MaskedOracleModel(cfg, sd, "sdpa_math").loss(ids, labels, attention_mask=mask)
    loss.backward()
    return float(loss), {k: v.grad for k, v in sd.items() if v.grad is not None}


@pytest.mark.parametrize("cfg", CFGS, ids=lambda c: c.name)
@pytest.mark.parametrize("kind", ["left", "right", "mixed"])
@pytest.mark.parametrize("n_mb,S", [(1, 48), (2, 48), (1, 700), (2, 700)], ids=["1", "2", "1-S700", "2-S700"])
def test_padded_step_vs_oracle_autograd(cfg, kind, n_mb, S):
    B = 4
    ids, mask, labels = padded(cfg, B, S, kind)
    loss32, g32 = _oracle_grads(cfg, ids, mask, labels, torch.float32)
    loss16, g16 = _oracle_grads(cfg, ids, mask, labels, torch.bfloat16)
    dm, opt = _dm(cfg, n_mb, B, S)
    opt.zero_grad()
    out = dm(ids, attention_mask=mask, labels=labels)
    out.loss.backward()
    torch.cuda.synchronize()
    print(f"{cfg.name} {kind} n_mb={n_mb} S={S}: loss gpu {float(out.loss):.6f} oracle_bf16 {loss16:.6f} "
          f"oracle_fp32 {loss32:.6f}")
    assert abs(float(out.loss) - loss32) <= max(2 * abs(loss16 - loss32), 2e-3)
    got = dm.stage.params.hf_state_dict(grads=True)
    names = ["model.layers.0.self_attn.q_norm.weight", "model.layers.2.self_attn.k_norm.weight",
             "model.layers.0.self_attn.k_proj.weight"] if cfg.qk_norm else ["model.layers.0.self_attn.k_proj.bias"]
    for name in names + ["model.layers.0.self_attn.q_proj.weight", "model.layers.1.self_attn.o_proj.weight",
                         "model.layers.2.mlp.gate_proj.weight", "model.layers.2.mlp.up_proj.weight",
                         "model.layers.3.mlp.down_proj.weight", "model.layers.0.input_layernorm.weight",
                         "model.layers.3.post_attention_layernorm.weight", "model.norm.weight",
                         "model.embed_tokens.weight"] + ([] if cfg.tied else ["lm_head.weight"]):
        e_ref = O.rel_l2(g16[name], g32[name])
        e_gpu = O.rel_l2(got[name].cpu(), g32[name])
        print(f"  {name}: gpu-vs-fp32 {e_gpu:.3e} oracle_bf16-vs-fp32 {e_ref:.3e}")
        assert e_gpu <= 1.5 * e_ref + 2e-3, name


@pytest.mark.parametrize("cfg", CFGS, ids=lambda c: c.name)
@pytest.mark.parametrize("n_mb,S", [(1, 48), (2, 700)], ids=["1", "2-S700"])
def test_pad_tokens_do_not_matter(cfg, n_mb, S):
    """Another pad id: the same loss, gradient arena and parameters after an Adam step, bit for bit.  The pad id's
    embedding gradient row is exactly 0 where the lm_head is not tied to the embedding (a tied lm_head gives every
    vocabulary row a gradient through the softmax)."""
    B = 4
    ids, mask, labels = padded(cfg, B, S, "mixed")
    pad = int(ids[mask == 0][0])
    other = (pad + 1) % cfg.vocab
    ids2 = ids.masked_fill(mask == 0, other)
    dm, opt = _dm(cfg, n_mb, B, S)
    la, ga, pa = _step(dm, opt, ids, mask, labels)
    if not cfg.tied:
        assert float(dm.stage.params.hf_state_dict(grads=True)["model.embed_tokens.weight"][pad].float().abs().sum()) == 0.0
    dm2, opt2 = _dm(cfg, n_mb, B, S)
    lb, gb, pb = _step(dm2, opt2, ids2, mask, labels)
    assert la == lb and torch.equal(ga, gb) and torch.equal(pa, pb)


@pytest.mark.parametrize("cfg", CFGS, ids=lambda c: c.name)
@pytest.mark.parametrize("n_mb,S", [(1, 48), (2, 700)], ids=["1", "2-S700"])
def test_mask_reaches_only_the_labels_when_right_padded(cfg, n_mb, S):
    """Right padding: the batch with its mask equals, bit for bit, the same batch without a mask whose labels carry
    -100 where the label rule puts it; an all-ones mask equals no mask."""
    B = 4
    ids, mask, labels = padded(cfg, B, S, "right")
    shift = mask_shift_labels(torch.nn.functional.pad(labels, (0, 1), value=-100)[:, 1:], mask)
    ruled = torch.cat([labels[:, :1], shift[:, :-1]], dim=1)
    dm, opt = _dm(cfg, n_mb, B, S)
    a = _step(dm, opt, ids, mask, labels)
    dm, opt = _dm(cfg, n_mb, B, S)
    b = _step(dm, opt, ids, None, ruled)
    assert a[0] == b[0] and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
    dm, opt = _dm(cfg, n_mb, B, S)
    c = _step(dm, opt, ids, torch.ones_like(mask), ids)
    dm, opt = _dm(cfg, n_mb, B, S)
    d = _step(dm, opt, ids, None, ids)
    assert c[0] == d[0] and torch.equal(c[1], d[1]) and torch.equal(c[2], d[2])


@pytest.mark.parametrize("cfg", CFGS, ids=lambda c: c.name)
@pytest.mark.parametrize("n_mb,S", [(1, 48), (2, 700)], ids=["1", "2-S700"])
def test_padded_steps_are_bit_reproducible(cfg, n_mb, S):
    B = 4
    ids, mask, labels = padded(cfg, B, S, "mixed")
    runs = [_dm(cfg, n_mb, B, S, seed=11) for _ in range(2)]
    for step in range(2):
        (la, ga, pa), (lb, gb, pb) = (_step(dm, opt, ids, mask, labels) for dm, opt in runs)
        assert la == lb and torch.equal(ga, gb) and torch.equal(pa, pb), step
        assert float(ga.float().abs().sum()) > 0


def test_bad_masks_raise():
    cfg = C.TINY_QWEN2_D128
    ids = synthetic_tokens(cfg, 2, 8)
    dm, _ = _dm(cfg, 1, 2, 8)
    with pytest.raises(NotImplementedError):
        dm(ids, attention_mask=torch.tensor([[1, 1, 0, 1, 1, 1, 1, 1], [1] * 8]), labels=ids)        # a hole
    with pytest.raises(ValueError):
        dm(ids, attention_mask=torch.tensor([[0] * 8, [1] * 8]), labels=ids)                          # an empty row
    with pytest.raises(ValueError):
        dm(ids, attention_mask=torch.ones(2, 7, dtype=torch.int64), labels=ids)                       # wrong shape
