"""Run under torchrun, one H100 per rank, any world size <= n_layers: greedy generation through a world-stage pipeline
with the decode hops on peer-mapped mailboxes must equal the NCCL send/recv path and the single-stage run."""
import os
import sys

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
    rank, world = dist.get_rank(), dist.get_world_size()
    cfg = C.TINY_QWEN2_D128
    res = {}
    rows = int(os.environ.get("RING_ROWS", "2"))          # rows per micro-batch: <= 3 GEMV path, above it the GEMM path
    dm = DistributedModel(cfg, training=False, n_pipelines=world, max_batch=rows * world, max_seq=96)
    ids = synthetic_tokens(cfg, rows * world, 16).cuda()
    gen = dm.generate(ids if rank == 0 else None, max_new_tokens=40)
    res["used_ring"] = getattr(dm, "_ring", None) is not None
    gen2 = dm.generate(ids if rank == 0 else None, max_new_tokens=40)        # counters reset between generations
    os.environ["TL_P2P"] = "nccl"
    gen_nccl = dm.generate(ids if rank == 0 else None, max_new_tokens=40)
    os.environ.pop("TL_P2P")
    res["repeatable"] = bool(torch.equal(gen, gen2))
    res["peer_vs_nccl"] = bool(torch.equal(gen, gen_nccl))
    res["wait_ms"] = float(dm._ring.wait_ns.item()) * 1e-6 if res["used_ring"] else None
    if rank == 0:
        single = DistributedModel(cfg, training=False, n_pipelines=world, max_batch=rows * world, max_seq=96, link=StageLink(0, 1))
        res["vs_single"] = bool(torch.equal(gen, single.generate(ids, max_new_tokens=40)))
    # checkpoint out of the sharded job (one safetensors file per stage + index), back into a single stage
    ck = os.path.join(out_dir, "ckpt")
    dm.save_pretrained(ck)
    res["ckpt_files"] = sorted(f for f in os.listdir(ck) if f.endswith(".safetensors"))
    if rank == 0:
        again = DistributedModel(ck, training=False, n_pipelines=world, max_batch=rows * world, max_seq=96, link=StageLink(0, 1), seed=5)
        res["ckpt_roundtrip"] = bool(torch.equal(gen, again.generate(ids, max_new_tokens=40)))
    torch.save(res, os.path.join(out_dir, f"ring{rank}.pt"))
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
