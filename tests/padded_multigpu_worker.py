"""Run under torchrun with one H100 per rank (NCCL): a padded training step pipelined over the ranks must equal the
single-stage step on rank 0's GPU bit for bit (same micro-batching, so the same kernels run on the same shapes)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tensorlink_b200.ml import DistributedModel  # noqa: E402
from tensorlink_b200.ml import configs as C  # noqa: E402
from tensorlink_b200.p2p.link import StageLink  # noqa: E402
from tests.test_train_padded_gpu import padded  # noqa: E402


def main(out_dir):
    dm = DistributedModel(C.TINY_QWEN2_D128, training=True, n_pipelines=2, max_batch=4, max_seq=128,
                          optimizer=torch.optim.Adam)
    rank = dm.rank
    ids, mask, labels = (t.cuda() for t in padded(C.TINY_QWEN2_D128, 4, 100, "mixed"))
    first = rank == 0
    o = dm(ids if first else None, attention_mask=mask if first else None, labels=labels if first else None)
    o.loss.backward()
    torch.save({"loss": float(o.loss), "grads": {k: v.cpu() for k, v in dm.stage.params.hf_state_dict(grads=True).items()}},
               os.path.join(out_dir, f"rank{rank}.pt"))
    if first:
        single = DistributedModel(C.TINY_QWEN2_D128, training=True, n_pipelines=2, max_batch=4, max_seq=128,
                                  link=StageLink(0, 1), optimizer=torch.optim.Adam)
        so = single(ids, attention_mask=mask, labels=labels)
        so.loss.backward()
        torch.save({"loss": float(so.loss),
                    "grads": {k: v.cpu() for k, v in single.stage.params.hf_state_dict(grads=True).items()}},
                   os.path.join(out_dir, "single.pt"))
    dm.link.barrier()


if __name__ == "__main__":
    try:
        main(sys.argv[1])
    except Exception:
        import traceback
        with open(os.path.join(sys.argv[1], f"err{os.environ.get('RANK', '0')}.txt"), "w") as f:
            traceback.print_exc(file=f)
        raise
