"""Run under torchrun with one H100 per rank (NCCL): a 2-stage FP8 pipeline must equal the single-stage FP8 model on
rank 0's GPU bit for bit (each stage holds its own FP8 layers; the last layer of stage 0 prefetches FP8 weights and its
down projection writes into the peer mailbox)."""
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

QC = {"quant_method": "fp8", "fmt": "e4m3", "activation_scheme": "dynamic", "weight_block_size": [128, 128]}


def main(out_dir):
    init_process_group_from_env("nccl")
    rank = dist.get_rank()
    cfg = C.TINY_QWEN2_D128
    kw = dict(training=False, n_pipelines=2, max_batch=4, max_seq=96, quantization_config=QC)
    single = DistributedModel(cfg, link=StageLink(0, 1), **kw) if rank == 0 else None
    dm = DistributedModel(cfg, **kw)
    ids = synthetic_tokens(cfg, 4, 20).cuda()
    res = {}
    out = dm(ids if rank == 0 else None, gather_logits=True)
    gen = dm.generate(ids if rank == 0 else None, max_new_tokens=24)
    gen_ng = dm.generate(ids if rank == 0 else None, max_new_tokens=24, use_graph=False)
    os.environ["TL_P2P"] = "nccl"
    gen_nccl = dm.generate(ids if rank == 0 else None, max_new_tokens=24)
    os.environ.pop("TL_P2P")
    if rank == 0:
        res["logits_equal"] = bool(torch.equal(out.logits, single(ids).logits))
        res["gen_equal"] = bool(torch.equal(gen, single.generate(ids, max_new_tokens=24)))
    res["gen_graph_vs_eager"] = bool(torch.equal(gen, gen_ng))
    res["gen_peer_vs_nccl"] = bool(torch.equal(gen, gen_nccl))
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
