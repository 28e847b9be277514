"""Run under torchrun with one H100 per rank (NCCL): a 2-stage Qwen3-MoE pipeline must equal the single-stage model on
rank 0's GPU bit for bit.  The last MoE layer of stage 0 stores its output straight into the next stage's peer-mapped
input: the expert GEMV's down launch in decode steps, the combine in prefill and batched decode."""
import os
import sys
import traceback

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tensorlink_b200.ml import DistributedModel  # noqa: E402
from tensorlink_b200.ml import configs as C  # noqa: E402
from tensorlink_b200.ml.weights import synthetic_tokens  # noqa: E402
from tensorlink_b200.p2p.link import StageLink, init_process_group_from_env  # noqa: E402


def main(out_dir):
    init_process_group_from_env("nccl")
    rank = dist.get_rank()
    cfg = C.TINY_QWEN3_MOE
    res = {}
    for B in (1, 8):                                  # the expert GEMV (decode) and the grouped path (batched decode)
        kw = dict(training=False, max_batch=B, max_seq=96)
        single = DistributedModel(cfg, link=StageLink(0, 1), **kw) if rank == 0 else None
        dm = DistributedModel(cfg, **kw)
        ids = synthetic_tokens(cfg, B, 20).cuda()
        out = dm(ids if rank == 0 else None, gather_logits=True)
        gen = dm.generate(ids if rank == 0 else None, max_new_tokens=16)
        gen_ng = dm.generate(ids if rank == 0 else None, max_new_tokens=16, use_graph=False)
        if rank == 0:
            res[f"logits_equal_B{B}"] = bool(torch.equal(out.logits, single(ids).logits))
            res[f"gen_equal_B{B}"] = bool(torch.equal(gen, single.generate(ids, max_new_tokens=16)))
        res[f"gen_graph_vs_eager_B{B}"] = bool(torch.equal(gen, gen_ng))
        del dm, single
    torch.save(res, os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    try:
        main(sys.argv[1])
    except Exception:
        with open(os.path.join(sys.argv[1], f"err{os.environ.get('RANK', '0')}.txt"), "w") as f:
            f.write(traceback.format_exc())
        raise
