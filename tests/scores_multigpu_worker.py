"""Run under torchrun, one H100 per rank: generate(return_dict_in_generate=True, output_scores=True, output_logits=True)
through a world-stage pipeline, greedy with logits processors and sampled, over the peer ring and over NCCL.  Every rank's
sequences, scores and logits must equal the single-stage run's bit for bit.  Writes sc<rank>.pt with the comparisons."""
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

NEW = 20
OUT = dict(return_dict_in_generate=True, output_scores=True, output_logits=True)
CASES = {"greedy": dict(repetition_penalty=1.3, no_repeat_ngram_size=2),
         "sampled": dict(do_sample=True, temperature=0.9, top_k=20, top_p=0.95, seed=5)}


def _flat(o):
    return o.sequences.cpu(), torch.stack(o.scores).cpu(), torch.stack(o.logits).cpu()


def main(out_dir):
    init_process_group_from_env("nccl")
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    cfg = C.TINY_QWEN2_D128
    rows = 2
    kw_model = dict(training=False, n_pipelines=world, max_batch=rows * world, max_seq=96)
    dm = DistributedModel(cfg, **kw_model)
    ids = synthetic_tokens(cfg, rows * world, 16).cuda()
    got = {}
    for transport in ("peer", "nccl"):
        if transport == "nccl":
            os.environ["TL_P2P"] = "nccl"
        for name, kw in CASES.items():
            got[(transport, name)] = _flat(dm.generate(ids if rank == 0 else None, max_new_tokens=NEW, **OUT, **kw))
        os.environ.pop("TL_P2P", None)
    single = DistributedModel(cfg, link=StageLink(0, 1), device=f"cuda:{torch.cuda.current_device()}", **kw_model)
    res = {"used_ring": getattr(dm, "_ring", None) is not None}
    for name, kw in CASES.items():
        want = _flat(single.generate(ids, max_new_tokens=NEW, **OUT, **kw))
        for transport in ("peer", "nccl"):
            res[f"{transport}_{name}"] = all(torch.equal(a, b) for a, b in zip(got[(transport, name)], want))
    torch.save(res, os.path.join(out_dir, f"sc{rank}.pt"))
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
