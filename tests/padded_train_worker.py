"""Run under torchrun (gloo, CPU): a padded training step through DistributedModel's multi-rank host logic with the
oracle stage twin that takes per-row key starts, against single-process autograd of the masked oracle."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import shard_oracle as O  # noqa: E402
from tensorlink_b200.ml import DistributedModel  # noqa: E402
from tensorlink_b200.ml import configs as C  # noqa: E402
from tensorlink_b200.ml.weights import init_state_dict, synthetic_tokens  # noqa: E402
from tensorlink_b200.p2p.link import init_process_group_from_env  # noqa: E402
from tests.padded_oracle import MaskedOracleModel, PaddedOracleStage  # noqa: E402


def padded_batch(cfg, B, S, seed=0):
    """ids, mask, labels: rows left-, right- and both-side padded (HF labels: -100 on pad positions)"""
    ids = synthetic_tokens(cfg, B, S, seed=seed)
    mask = torch.zeros(B, S, dtype=torch.int64)
    spans = [(3, S), (0, S - 5), (2, S - 4), (0, S)]
    for r in range(B):
        a, e = spans[r % len(spans)]
        mask[r, a:e] = 1
    ids = ids.masked_fill(mask == 0, 7)
    return ids, mask, ids.masked_fill(mask == 0, -100)


def main(out_dir):
    torch.set_num_threads(2)
    init_process_group_from_env("gloo")
    rank = dist.get_rank()
    cfg = C.TINY_QWEN2_D128
    sd = init_state_dict(cfg)
    ids, mask, labels = padded_batch(cfg, 4, 16)
    dm = DistributedModel(cfg, training=True, n_pipelines=2, max_batch=4, max_seq=64, _stage_factory=PaddedOracleStage,
                          device="cpu", optimizer=torch.optim.Adam)
    first = rank == 0
    o = dm(ids if first else None, attention_mask=mask if first else None, labels=labels if first else None)
    o.loss.backward()
    ref_sd = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    ref_loss, _ = MaskedOracleModel(cfg, ref_sd, "sdpa_math").loss(ids, labels, attention_mask=mask)
    ref_loss.backward()
    res = {"loss_close": abs(float(o.loss) - float(ref_loss)) < 2e-3}
    worst = 0.0
    for k, v in dm.stage.sd.items():
        if v.grad is not None and ref_sd[k].grad is not None:
            worst = max(worst, O.rel_l2(v.grad, ref_sd[k].grad))
    res["grad_worst_rel_l2"] = worst
    res["n_params_with_grad"] = sum(v.grad is not None for v in dm.stage.sd.values())
    torch.save(res, os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    try:
        main(sys.argv[1])
    except Exception:
        import traceback
        with open(os.path.join(sys.argv[1], f"err{os.environ.get('RANK', '0')}.txt"), "w") as f:
            traceback.print_exc(file=f)
        raise
