"""Run under torchrun, one H100 per rank: generation with repetition_penalty / no_repeat_ngram_size / min_new_tokens
through a world-stage pipeline, greedy and sampled, with the decode hops on peer-mapped mailboxes and over NCCL, must
equal the single-stage run bit for bit.  Writes lp<rank>.pt with the comparisons."""
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

NEW = 24


def main(out_dir):
    init_process_group_from_env("nccl")
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))    # (no group at world 1)
    cfg = C.TINY_QWEN2_D128
    rows = 2                                   # rows per micro-batch (GEMV path), one micro-batch per stage
    kw_model = dict(training=False, n_pipelines=world, max_batch=rows * world, max_seq=96)
    dm = DistributedModel(cfg, **kw_model)
    ids = synthetic_tokens(cfg, rows * world, 16).cuda()
    plain = dm.generate(ids if rank == 0 else None, max_new_tokens=NEW)
    eos = int(plain[0, 16 + 1])                # emitted at the second step without the processors
    procs = dict(repetition_penalty=1.3, no_repeat_ngram_size=2, min_new_tokens=6, eos_token_id=eos, pad_token_id=0)
    cases = {"greedy": procs, "sampled": dict(procs, do_sample=True, temperature=0.9, top_k=20, top_p=0.95, seed=5)}
    out = {}
    for transport in ("peer", "nccl"):
        if transport == "nccl":
            os.environ["TL_P2P"] = "nccl"
        for name, kw in cases.items():
            out[(transport, name)] = dm.generate(ids if rank == 0 else None, max_new_tokens=NEW, **kw).cpu()
        os.environ.pop("TL_P2P", None)
    res = {"used_ring": getattr(dm, "_ring", None) is not None}
    for name in cases:
        res[f"{name}_peer_vs_nccl"] = bool(torch.equal(out[("peer", name)], out[("nccl", name)]))
        res[f"{name}_min_new_held"] = all(eos not in r[16:16 + 6].tolist() for r in out[("peer", name)])
    res["sampled_differs"] = not torch.equal(out[("peer", "greedy")], out[("peer", "sampled")])
    if rank == 0:
        single = DistributedModel(cfg, link=StageLink(0, 1), **kw_model)
        for name, kw in cases.items():
            res[f"{name}_vs_single"] = bool(torch.equal(out[("peer", name)], single.generate(ids, max_new_tokens=NEW, **kw).cpu()))
    torch.save(res, os.path.join(out_dir, f"lp{rank}.pt"))
    if dist.is_initialized():
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
