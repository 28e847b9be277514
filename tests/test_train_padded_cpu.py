"""Padded training batches on the CPU: the attention_mask parsing of the training forward, the label rule, the masked
oracle against the installed HF implementation, and a padded step through 2 and 3 gloo ranks."""
import os
import socket
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from tensorlink_b200.ml import configs as C
from tensorlink_b200.ml import module as M
from tensorlink_b200.ml.weights import init_state_dict
from tests.hf_util import hf_model
from tests.padded_oracle import MaskedOracleModel, mask_shift_labels
from tests.padded_train_worker import padded_batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_train_mask_parsing():
    assert M._train_mask(None, (2, 4)) is None
    assert M._train_mask(torch.ones(2, 4), (2, 4)) is None
    starts, real = M._train_mask(torch.tensor([[0, 0, 1, 1], [1, 1, 1, 0], [0, 1, 1, 0], [1, 1, 1, 1]]), (4, 4))
    assert starts == [2, 0, 1, 0]
    assert real.dtype == torch.bool and torch.equal(real.long(), torch.tensor([[0, 0, 1, 1], [1, 1, 1, 0], [0, 1, 1, 0],
                                                                               [1, 1, 1, 1]]))
    starts, _ = M._train_mask(torch.tensor([[0, 0, 0, 1]]), (1, 4))          # one real token
    assert starts == [3]
    with pytest.raises(NotImplementedError):
        M._train_mask(torch.tensor([[1, 0, 1, 1]]), (1, 4))                    # a hole
    with pytest.raises(ValueError):
        M._train_mask(torch.tensor([[0, 0, 0, 0], [1, 1, 1, 1]]), (2, 4))      # a row without a real token
    with pytest.raises(ValueError):
        M._train_mask(torch.ones(2, 5), (2, 4))                                # shaped unlike input_ids


def test_label_rule():
    labels = torch.tensor([[-100, -100, 5, 6, 7], [1, 2, 3, -100, -100]])
    mask = torch.tensor([[0, 0, 1, 1, 1], [1, 1, 1, 0, 0]])
    shift = F.pad(labels, (0, 1), value=-100)[:, 1:]
    got = mask_shift_labels(shift, mask)
    # left padding: the first real token (5) is no longer predicted from the last pad; right padding: unchanged
    assert torch.equal(got, torch.tensor([[-100, -100, 6, 7, -100], [2, 3, -100, -100, -100]]))
    assert torch.equal(mask_shift_labels(shift, None), shift)


def _hf_reference(cfg, sd, attn, ids, mask, labels, dtype):
    hf = hf_model(cfg, sd, attn, dtype)
    with torch.no_grad():
        logits = hf(input_ids=ids, attention_mask=mask).logits
        shift = mask_shift_labels(F.pad(labels, (0, 1), value=-100)[:, 1:], mask)
        hf_labels = torch.cat([labels[:, :1], shift[:, :-1]], dim=1)          # HF shifts these back to ``shift``
        loss = hf(input_ids=ids, attention_mask=mask, labels=hf_labels).loss
    return logits, loss


@pytest.mark.parametrize("cfg", [C.TINY_QWEN2, C.TINY_QWEN2_D128, C.TINY_QWEN3], ids=lambda c: c.name)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_masked_oracle_bit_exact_vs_hf_eager(cfg, dtype):
    """Real positions of a left-, right- and both-side padded batch: logits and the rule-masked loss equal HF eager's
    bit for bit (HF forward without position_ids: positions 0..S-1 in every row)."""
    sd = init_state_dict(cfg, dtype=dtype)
    ids, mask, labels = padded_batch(cfg, 4, 24, seed=3)
    ref, ref_loss = _hf_reference(cfg, sd, "eager", ids, mask, labels, dtype)
    with torch.no_grad():
        got = MaskedOracleModel(cfg, sd, "eager").logits(ids, attention_mask=mask)
        got3 = MaskedOracleModel(cfg, sd, "eager").logits(ids, n_shards=3, attention_mask=mask)
        loss, _ = MaskedOracleModel(cfg, sd, "eager").loss(ids, labels, attention_mask=mask)
    real = mask.bool()
    assert torch.equal(got[real], ref[real])
    assert torch.equal(got3[real], ref[real])
    assert torch.equal(loss, ref_loss)


@pytest.mark.parametrize("cfg", [C.TINY_QWEN2, C.TINY_QWEN2_D128, C.TINY_QWEN3], ids=lambda c: c.name)
def test_masked_oracle_sdpa_math_close_to_hf_sdpa(cfg):
    """As tests/test_oracle_vs_hf.py for unpadded batches: 'sdpa_math' vs HF sdpa on the real positions, relative to
    the spread between HF's own eager and sdpa paths."""
    from oracle import shard_oracle as O
    sd = init_state_dict(cfg)
    ids, mask, labels = padded_batch(cfg, 4, 40, seed=4)
    ref, ref_loss = _hf_reference(cfg, sd, "sdpa", ids, mask, labels, torch.bfloat16)
    ref_e, _ = _hf_reference(cfg, sd, "eager", ids, mask, labels, torch.bfloat16)
    with torch.no_grad():
        got = MaskedOracleModel(cfg, sd, "sdpa_math").logits(ids, attention_mask=mask)
        loss, _ = MaskedOracleModel(cfg, sd, "sdpa_math").loss(ids, labels, attention_mask=mask)
    real = mask.bool()
    floor = O.rel_l2(ref_e[real], ref[real])
    assert O.rel_l2(got[real], ref[real]) <= 1.25 * floor, (O.rel_l2(got[real], ref[real]), floor)
    assert abs(float(loss) - float(ref_loss)) <= 2e-2


def test_unpadded_mask_is_the_plain_oracle():
    cfg = C.TINY_QWEN2
    sd = init_state_dict(cfg)
    ids, _, _ = padded_batch(cfg, 2, 12)
    with torch.no_grad():
        a = MaskedOracleModel(cfg, sd).logits(ids, attention_mask=torch.ones_like(ids))
        b = MaskedOracleModel(cfg, sd).logits(ids)
    assert torch.equal(a, b)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.parametrize("world", [2, 3])
def test_padded_training_across_gloo_ranks(tmp_path, world):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
           "127.0.0.1", "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "padded_train_worker.py"),
           str(tmp_path)]
    env = dict(os.environ, OMP_NUM_THREADS="2", PYTHONPATH=ROOT)
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    errs = "".join(open(p).read() for p in sorted(map(str, tmp_path.glob("err*.txt"))))
    assert r.returncode == 0, errs or r.stderr[-3000:]
    for i in range(world):
        res = torch.load(tmp_path / f"rank{i}.pt")
        assert res["loss_close"]
        # bf16 autograd in pieces (a gradient crossing a rank boundary is rounded to bf16 once more) vs one graph
        assert res["grad_worst_rel_l2"] < 2e-2 and res["n_params_with_grad"] >= 3
