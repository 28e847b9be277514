"""Left-padded batches through ``DistributedModel.generate`` as ONE batch: one prefill per micro-batch, one decode loop.

Each row must give the tokens of its own prompt generated alone, unpadded: the float oracle's greedy tokens wherever the
oracle's top-2 margin is >= 0.05 (up to the first closer call), and ``dm.generate`` on that row alone on the same
steps.  Cases cover the GEMV (2-3 rows) and GEMM (4-8 rows) decode paths, the fused (max_seq <= 2048) and split-KV
(> 2048) decode attention, one and two micro-batches, and eager and graph-captured decode.
"""
import pytest
import torch

from oracle import shard_oracle as O
from tensorlink_b200.ml import configs as C
from tensorlink_b200.ml import module as M
from tensorlink_b200.ml.weights import init_state_dict, synthetic_tokens

pytestmark = pytest.mark.gpu

MARGIN = 0.05
PAD = 0

CASES = [  # cfg, lengths of the rows, max_seq, n_pipelines, use_graph
    ("TINY_QWEN2", (5, 17, 11), 256, 1, True),
    ("TINY_QWEN3", (9, 1, 30), 2304, 1, False),
    ("TINY_QWEN2_D128", (70, 3), 256, 1, False),
    ("TINY_QWEN2_D128", (12, 40, 7, 66, 25, 3), 2304, 1, True),
    ("TINY_QWEN3", (8, 21, 64, 65, 2, 33, 17, 50), 256, 2, True),
    ("TINY_QWEN2", (31, 4, 19, 64), 2304, 2, False),
    ("TINY_QWEN2", (6, 13, 20, 27, 34, 41, 48, 55), 256, 1, False),
]
NEW = 12


def _batch(cfg, lengths, lead=0):
    """Left-padded ids / mask for rows of the given real lengths (+ `lead` columns of padding in every row)."""
    S = max(lengths) + lead
    ids = torch.full((len(lengths), S), PAD, dtype=torch.int64)
    mask = torch.zeros(len(lengths), S, dtype=torch.int64)
    rows = []
    for b, L in enumerate(lengths):
        r = synthetic_tokens(cfg, 1, L, seed=17 + b)
        ids[b, S - L:] = r[0]
        mask[b, S - L:] = 1
        rows.append(r)
    return ids, mask, rows


def _model(cfg, max_seq, n_pipelines, B):
    from tensorlink_b200.ml import DistributedModel
    return DistributedModel(cfg, training=False, max_batch=max(B, n_pipelines), max_seq=max_seq, n_pipelines=n_pipelines)


class Streamer:
    def __init__(self):
        self.cols, self.ended = [], False

    def put(self, t):
        self.cols.append(t.clone())

    def end(self):
        self.ended = True


@pytest.mark.parametrize("name,lengths,max_seq,n_pipelines,use_graph", CASES)
def test_padded_batch_matches_rows_alone(name, lengths, max_seq, n_pipelines, use_graph):
    cfg = getattr(C, name)
    sd = init_state_dict(cfg)
    dm = _model(cfg, max_seq, n_pipelines, len(lengths))
    ids, mask, rows = _batch(cfg, lengths)
    B, S = ids.shape
    calls = []
    prefill = dm.stage.prefill
    dm.stage.prefill = lambda *a, **k: (calls.append(k.get("kv_start")), prefill(*a, **k))[1]
    streamer = Streamer()
    got = dm.generate(ids, attention_mask=mask, max_new_tokens=NEW, use_graph=use_graph, streamer=streamer).cpu()
    dm.stage.prefill = prefill
    n_mb = n_pipelines if B % n_pipelines == 0 else 1
    assert len(calls) == n_mb and all(c is not None for c in calls), calls        # one prefill per micro-batch
    assert got.shape == (B, S + NEW) and torch.equal(got[:, :S], ids)
    assert streamer.ended and len(streamer.cols) == NEW
    assert torch.equal(torch.stack(streamer.cols, 1), got[:, S:])                   # every column of every row
    oracle = O.OracleModel(cfg, sd, "sdpa_math")
    for b, r in enumerate(rows):
        want, margins = oracle.generate(r, NEW, return_margins=True)
        alone = dm.generate(r, max_new_tokens=NEW, use_graph=use_graph).cpu()
        L = r.shape[1]
        for s in range(NEW):
            if margins[0, s] < MARGIN:
                break
            assert int(got[b, S + s]) == int(want[0, L + s]), (b, s, got[b, S:], want[0, L:])
            assert int(got[b, S + s]) == int(alone[0, L + s]), (b, s, got[b, S:], alone[0, L:])


def test_padded_eos_trim_and_sampling():
    cfg = C.TINY_QWEN2_D128
    dm = _model(cfg, 256, 1, 4)
    lengths = (7, 30, 12, 19)
    ids, mask, _ = _batch(cfg, lengths)
    S = ids.shape[1]
    base = dm.generate(ids, attention_mask=mask, max_new_tokens=40).cpu()
    # EOS: a token row 0 emits early; every row's tail after its first EOS becomes pad, and the run stops early
    eos = int(base[0, S + 2])
    got = dm.generate(ids, attention_mask=mask, max_new_tokens=40, eos_token_id=eos, pad_token_id=PAD).cpu()
    assert torch.equal(got, M.apply_eos(base, S, eos, PAD))
    # columns that are pad in every row are dropped before the run and return in the result
    ids3, mask3, _ = _batch(cfg, lengths, lead=3)
    got3 = dm.generate(ids3, attention_mask=mask3, max_new_tokens=40).cpu()
    assert torch.equal(got3[:, :3], ids3[:, :3]) and torch.equal(got3[:, 3:], base)
    assert M._left_pad_starts(mask3) == (3, [S - L for L in lengths])
    # a seeded sampling call reproduces its tokens
    kw = dict(attention_mask=mask, max_new_tokens=20, do_sample=True, temperature=0.9, top_k=20, seed=123)
    a, b = dm.generate(ids, **kw).cpu(), dm.generate(ids, **kw).cpu()
    assert torch.equal(a, b)
