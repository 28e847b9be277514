"""Run under torchrun, one H100 per rank: sampled generation with min_p / typical_p / epsilon_cutoff / eta_cutoff
through a world-stage pipeline must equal the single-stage run bit for bit (the sampling dict reaches the last stage,
which draws), and min_p = 1 / epsilon_cutoff near 1 must reproduce greedy decoding's tokens.  Writes wp<rank>.pt."""
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

NEW = 16
SAMPLE = dict(do_sample=True, temperature=0.9, top_k=0, seed=5)
CASES = {"chain": dict(SAMPLE, min_p=0.02, typical_p=0.9, epsilon_cutoff=1e-4, eta_cutoff=5e-4),
         "chain_procs": dict(SAMPLE, min_p=0.02, typical_p=0.9, eta_cutoff=5e-4, repetition_penalty=1.3,
                             no_repeat_ngram_size=2),
         "min_p1": dict(SAMPLE, min_p=1.0), "eps_sharp": dict(SAMPLE, epsilon_cutoff=0.999999)}


def main(out_dir):
    init_process_group_from_env("nccl")
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    cfg = C.TINY_QWEN2_D128
    rows = 2
    kw_model = dict(training=False, n_pipelines=world, max_batch=rows * world, max_seq=96)
    dm = DistributedModel(cfg, **kw_model)
    ids = synthetic_tokens(cfg, rows * world, 16).cuda()
    g = dm.generate(ids if rank == 0 else None, max_new_tokens=NEW, return_dict_in_generate=True, output_logits=True)
    greedy = g.sequences.cpu()
    # the sharp settings keep only the top token: greedy's tokens wherever no step has a top-2 tie
    no_tie = all(bool((torch.topk(lg.float(), 2, dim=-1).values.diff(dim=-1) < 0).all()) for lg in g.logits)
    out = {name: dm.generate(ids if rank == 0 else None, max_new_tokens=NEW, **kw).cpu() for name, kw in CASES.items()}
    res = {"sharp_is_greedy": not no_tie or all(torch.equal(out[n], greedy) for n in ("min_p1", "eps_sharp")),
           "chain_differs": not torch.equal(out["chain"], greedy)}
    if rank == 0:
        single = DistributedModel(cfg, link=StageLink(0, 1), **kw_model)
        res["single_greedy_equal"] = bool(torch.equal(single.generate(ids, max_new_tokens=NEW).cpu(), greedy))
        for name, kw in CASES.items():
            res[f"{name}_vs_single"] = bool(torch.equal(out[name], single.generate(ids, max_new_tokens=NEW, **kw).cpu()))
    torch.save(res, os.path.join(out_dir, f"wp{rank}.pt"))
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
