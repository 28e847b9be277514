"""Run under torchrun with one H100 per rank (NCCL): pipeline-sharded results must equal the single-stage results
computed with the same kernels on rank 0's GPU (sharding must not change a bit: same launches, same order)."""
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
    # same micro-batching as the pipeline (2 x 2 rows), so the same kernels run on the same shapes
    single = DistributedModel(cfg, training=False, n_pipelines=2, max_batch=4, max_seq=96, link=StageLink(0, 1)) if rank == 0 else None
    dm = DistributedModel(cfg, training=False, n_pipelines=2, max_batch=4, max_seq=96)
    ids = synthetic_tokens(cfg, 4, 20).cuda()
    out = dm(ids if rank == 0 else None, gather_logits=True)
    gen = dm.generate(ids if rank == 0 else None, max_new_tokens=24)
    gen_ng = dm.generate(ids if rank == 0 else None, max_new_tokens=24, use_graph=False)
    if rank == 0:
        ref_logits = single(ids).logits
        ref_gen = single.generate(ids, max_new_tokens=24)
        res["logits_equal"] = bool(torch.equal(out.logits, ref_logits))
        res["gen_equal"] = bool(torch.equal(gen, ref_gen))
    res["gen_graph_vs_eager"] = bool(torch.equal(gen, gen_ng))
    # the two generations above hopped over peer-mapped mailboxes (p2p/peer.py); NCCL send/recv must give the same ids
    res["used_ring"] = getattr(dm, "_ring", None) is not None
    os.environ["TL_P2P"] = "nccl"
    gen_nccl = dm.generate(ids if rank == 0 else None, max_new_tokens=24)
    os.environ.pop("TL_P2P")
    res["gen_peer_vs_nccl"] = bool(torch.equal(gen, gen_nccl))

    # EOS early stop on both transports: 40 tokens requested, the token the model emits at step 2 of row 0 declared EOS for a
    # one-row-per-micro-batch run -> every rank returns the same, shortened result as the single stage does
    ids2 = ids[[0, 0]].contiguous()         # two copies of row 0: both finish at step 2, the loop stops at its next check
    eos = int(gen[0, 20 + 2])
    for tag, env in (("peer", None), ("nccl", "nccl")):
        if env:
            os.environ["TL_P2P"] = env
        got = dm.generate(ids2 if rank == 0 else None, max_new_tokens=40, eos_token_id=eos, pad_token_id=0)
        if env:
            os.environ.pop("TL_P2P")
        res[f"eos_{tag}_shape"] = tuple(got.shape)
        if rank == 0:
            want = single.generate(ids2, max_new_tokens=40, eos_token_id=eos, pad_token_id=0)
            res[f"eos_{tag}_equal"] = bool(got.shape == want.shape and torch.equal(got, want) and got.shape[1] < 60)

    class Cols:
        def __init__(self):
            self.cols, self.ended = [], False

        def put(self, t):
            self.cols.append(t.clone())

        def end(self):
            self.ended = True

    sink = Cols()
    gen_s = dm.generate(ids if rank == 0 else None, max_new_tokens=6, streamer=sink)
    if rank == 0:
        res["stream_ok"] = bool(sink.ended and len(sink.cols) == 6 and
                                torch.equal(torch.stack(sink.cols, 1).cuda(), gen_s[:, 20:]) and torch.equal(gen_s, gen[:, :26]))
    res["bytes_sent_infer"] = dm.link.bytes_sent
    # training: 2 micro-batches through the 2 stages
    tids = synthetic_tokens(cfg, 4, 32).cuda()
    dmt = DistributedModel(cfg, training=True, n_pipelines=2, max_batch=4, max_seq=64, optimizer=torch.optim.Adam)
    opt = dmt.create_optimizer(lr=1e-3)
    opt.zero_grad()
    o = dmt(tids if rank == 0 else None, labels=tids if rank == 0 else None)
    o.loss.backward()
    grads = {k: v.cpu() for k, v in dmt.stage.params.hf_state_dict(grads=True).items()}
    opt.step()
    res["loss"] = float(o.loss)
    if rank == 0:
        st = DistributedModel(cfg, training=True, n_pipelines=2, max_batch=4, max_seq=64, link=StageLink(0, 1),
                              optimizer=torch.optim.Adam)
        so = st(tids, labels=tids)
        so.loss.backward()
        ref = {k: v.cpu() for k, v in st.stage.params.hf_state_dict(grads=True).items()}
        res["loss_single"] = float(so.loss)
        torch.save(ref, os.path.join(out_dir, "ref_grads.pt"))
    # tied embeddings split over the two ranks (Qwen2.5-0.5B layout): both copies must end up with the summed gradient
    tc = C.TINY_QWEN2
    tt = synthetic_tokens(tc, 2, 24).cuda()
    dtie = DistributedModel(tc, training=True, n_pipelines=1, max_batch=2, max_seq=32, optimizer=torch.optim.Adam)
    ot = dtie(tt if rank == 0 else None, labels=tt if rank == 0 else None)
    ot.loss.backward()
    key = "embed" if rank == 0 else "head"
    torch.save(dtie.stage.params.g[key].cpu(), os.path.join(out_dir, f"tied{rank}.pt"))
    if rank == 0:
        s1 = DistributedModel(tc, training=True, n_pipelines=1, max_batch=2, max_seq=32, link=StageLink(0, 1),
                              optimizer=torch.optim.Adam)
        s1(tt, labels=tt).loss.backward()
        torch.save(s1.stage.params.g["embed"].cpu(), os.path.join(out_dir, "tied_ref.pt"))
    # gradient accumulation on the tied split: a second backward without zero_grad must add ITS delta once on both copies
    ot2 = dtie(tt if rank == 0 else None, labels=tt if rank == 0 else None)
    ot2.loss.backward()
    torch.save(dtie.stage.params.g[key].cpu(), os.path.join(out_dir, f"tied2_{rank}.pt"))
    if rank == 0:
        s1(tt, labels=tt).loss.backward()
        torch.save(s1.stage.params.g["embed"].cpu(), os.path.join(out_dir, "tied2_ref.pt"))
    # the same with two micro-batches: deferred weight gradients and the split head backward (the lm_head gradient exists only
    # after the stage's weight-gradient phase, and is exchanged then)
    dtie2 = DistributedModel(tc, training=True, n_pipelines=2, max_batch=2, max_seq=32, optimizer=torch.optim.Adam)
    dtie2(tt if rank == 0 else None, labels=tt if rank == 0 else None).loss.backward()
    res["tied_split_head"] = bool(dtie2.stage.trainer.head_split) if rank == 1 else None
    torch.save(dtie2.stage.params.g[key].cpu(), os.path.join(out_dir, f"tied3_{rank}.pt"))
    torch.save(grads, os.path.join(out_dir, f"grads{rank}.pt"))
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
