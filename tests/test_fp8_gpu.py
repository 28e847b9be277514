"""FP8 weights on the H100: the FP8 GEMV and the dequantization kernel element by element, and FP8 models against the
bf16 model built from HF's dequantized weights, bit for bit on every decode path."""
from dataclasses import replace

import pytest
import torch

from oracle import shard_oracle as O
from tests import linear_cases as L
from tensorlink_b200 import native as nat
from tensorlink_b200.ml import DistributedModel
from tensorlink_b200.ml import configs as C
from tensorlink_b200.ml import fp8 as F8
from tensorlink_b200.ml.shard import fp8_gemv_max_rows
from tensorlink_b200.ml.weights import synthetic_tokens

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _release_memory():
    """The model tests hold several models at once: hand their memory back before the next test."""
    yield
    import gc
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


QC = {"quant_method": "fp8", "fmt": "e4m3", "activation_scheme": "dynamic", "weight_block_size": [128, 128]}
DEV = "cuda"


def _fp8_linear(N, K, seed, std=0.02):
    """N rows of an FP8 weight quantized by HF's rule (row count rounded up to a block, then cut)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    R = (N + 127) // 128 * 128
    q, inv = F8.quantize(torch.randn(R, K, generator=g, device=DEV).mul_(std).to(torch.bfloat16))
    return q[:N].contiguous(), F8.rows_from_grid(inv)[:N].contiguous()


def _rand(shape, seed, std=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(*shape, generator=g, device=DEV).mul_(std).to(torch.bfloat16)


def test_dequant_equals_cpu():
    for N, K in ((256, 128), (384, 3584), (1024, 18944)):
        q, rows = _fp8_linear(N, K, N + K)
        got = nat.dequant_fp8(q, rows).cpu()
        want = F8.dequantize(q.cpu(), rows.cpu()[::128])
        assert torch.equal(got, want), (N, K)
        # a larger scratch buffer: only its first N*K elements are written
        scratch = torch.full((N * K + 1000,), 7.0, dtype=torch.bfloat16, device=DEV)
        assert torch.equal(nat.dequant_fp8(q, rows, out=scratch).cpu(), want)
        assert bool((scratch[N * K:] == 7.0).all())


def test_gemv_fp8_exact_integers():
    """Integer e4m3 codes, power-of-two scales and small integer activations: every product and partial sum is exact
    in fp32, so the result is the float64 product rounded once to bf16."""
    N, K = 512, 4096 + 128
    g = torch.Generator(device=DEV).manual_seed(3)
    codes = torch.randint(-8, 9, (N, K), generator=g, device=DEV).float()
    q = codes.to(torch.float8_e4m3fn)
    exps = torch.randint(-6, 1, (N, K // 128), generator=g, device=DEV).float()
    rows = torch.exp2(exps).contiguous()
    for M in (1, 2, 3, 4, 8):
        x = torch.randint(-3, 4, (M, K), generator=g, device=DEV).to(torch.bfloat16)
        y = nat.gemv_fp8(x, q, rows)
        w = codes.double() * torch.exp2(exps.double()).repeat_interleave(128, dim=1)
        want = (x.double() @ w.T).to(torch.bfloat16)
        assert torch.equal(y, want), M


SHAPES = [(2, 128), (6, 1024), (896, 896), (1152, 896), (3584, 3584), (2 * 4864, 896), (896, 4864), (3584, 8192),
          (3584, 8192 + 128), (512, 18944), (4608, 4096)]
# down projections of 32B / 72B models: x of 3 rows leaves the weight-streaming ring too few stages, so both GEMVs take
# the register-streaming kernel
WIDE = [(1024, 25600), (1024, 27648), (1024, 29568)]


@pytest.mark.parametrize("N,K", SHAPES)
def test_gemv_fp8_equals_bf16_over_dequant(N, K):
    """tl_gemv_fp8 == tl_gemv_bf16 over tl_dequant_fp8's output, bit for bit, for 1..8 rows and every epilogue; K and N
    straddle the stage (16 KB), chunk (8192 FP8 / 4096 bf16 columns) and ticket sizes."""
    q, rows = _fp8_linear(N, K, N * 7 + K)
    wb = nat.dequant_fp8(q, rows)
    norm = _rand((K,), 1, 0.5) + 1
    bias = _rand((N,), 2, 0.1)
    for M in range(1, 9):
        x = _rand((M, K), 10 + M)
        res = _rand((M, N), 20 + M)
        for kw in ({}, {"norm_w": norm}, {"bias": bias}, {"residual": res}, {"flags": nat.EPI_SWIGLU, "norm_w": norm},
                   {"bias": bias, "residual": res, "norm_w": norm}):
            got = nat.gemv_fp8(x, q, rows, **kw)
            want = nat.gemv(x, wb, **kw)
            assert torch.equal(got, want), (M, list(kw))


@pytest.mark.parametrize("N,K", WIDE)
def test_gemv_fp8_wide_k_equals_bf16_over_dequant(N, K):
    q, rows = _fp8_linear(N, K, K)
    wb = nat.dequant_fp8(q, rows)
    res = _rand((3, N), 5)
    for M in (1, 2, 3):
        x = _rand((M, K), 30 + M)
        for kw in ({}, {"residual": res[:M]}):
            assert torch.equal(nat.gemv_fp8(x, q, rows, **kw), nat.gemv(x, wb, **kw)), (M, list(kw))


def test_gemv_fp8_register_kernel_runs():
    q, rows = _fp8_linear(1024, 27648, 1)
    x = _rand((3, 27648), 2)
    nat.gemv_fp8(x, q, rows)
    torch.cuda.synchronize()
    with L.KernelLog() as log:
        nat.gemv_fp8(x, q, rows)
    assert [k.split("<")[0] for k, _ in log.kernels] == ["gemv_fp8_kernel"], log.all_names


def test_gemv_fp8_kernel_runs():
    q, rows = _fp8_linear(3584, 3584, 9)
    x = _rand((1, 3584), 4)
    nat.gemv_fp8(x, q, rows)
    torch.cuda.synchronize()
    with L.KernelLog() as log:
        nat.gemv_fp8(x, q, rows)
        nat.dequant_fp8(q, rows)
    assert [k for k, _ in log.kernels] == ["gemv_stream_fp8_kernel<1>", "dequant_fp8_kernel"], log.all_names


# ---------------------------------------------------------------------------------------------- model level
def _pair(cfg, max_batch=32, max_seq=128, init="seeded", seed=1234):
    """The FP8 model (quantized on load) and the bf16 model over its dequantized weights.  The bf16 model's layers take
    the FP8 model's GEMV row threshold, so both run the same Linear kernels at every row count."""
    f = DistributedModel(cfg, training=False, max_batch=max_batch, max_seq=max_seq, init=init, seed=seed,
                         quantization_config=QC)
    sd = f.state_dict()
    deq = {}
    for k, t in sd.items():
        if k.endswith("weight_scale_inv"):
            continue
        deq[k] = F8.dequantize(t, sd[k[:-len("weight")] + "weight_scale_inv"]) if t.dtype == torch.float8_e4m3fn else t
    b = DistributedModel(cfg, training=False, max_batch=max_batch, max_seq=max_seq, init=init, seed=seed)
    b.stage.params.load_hf_state_dict(deq)
    for g in b.stage.slots:
        g.gemv_rows = fp8_gemv_max_rows
    return f, b, deq


TINY = [C.TINY_QWEN2, C.TINY_QWEN2_D128, C.TINY_QWEN3]


@pytest.mark.parametrize("cfg", TINY, ids=lambda c: c.name)
def test_model_equals_bf16_over_dequantized(cfg):
    f, b, deq = _pair(cfg)
    for B in (1, 3, 8, 32):
        ids = synthetic_tokens(cfg, B, 12, seed=B)
        assert torch.equal(f(ids).logits, b(ids).logits), B
        assert torch.equal(f.generate(ids, max_new_tokens=10), b.generate(ids, max_new_tokens=10)), B
    ids = synthetic_tokens(cfg, 3, 12, seed=5)
    mask = torch.ones_like(ids)
    mask[0, :4] = 0
    mask[2, :7] = 0
    assert torch.equal(f.generate(ids, attention_mask=mask, max_new_tokens=8),
                       b.generate(ids, attention_mask=mask, max_new_tokens=8))
    kw = dict(max_new_tokens=12, do_sample=True, temperature=0.9, top_k=20, seed=7)
    assert torch.equal(f.generate(ids[:2], **kw), b.generate(ids[:2], **kw))
    kw = dict(max_new_tokens=12, repetition_penalty=1.3, no_repeat_ngram_size=2)
    assert torch.equal(f.generate(ids, **kw), b.generate(ids, **kw))
    one = synthetic_tokens(cfg, 1, 24, seed=9)
    one[0, 12:] = one[0, :12]
    assert torch.equal(f.generate(one, max_new_tokens=16, prompt_lookup_num_tokens=5),
                       b.generate(one, max_new_tokens=16, prompt_lookup_num_tokens=5))
    # the multi-pass FP8 GEMV (5..8 rows in passes of at most 4) against the bf16 GEMV in the same passes
    for m in (f, b):
        for g in m.stage.slots:
            g.gemv_rows = lambda: 8
    for B in (6, 8):
        ids8 = synthetic_tokens(cfg, B, 12, seed=B)
        assert torch.equal(f.generate(ids8, max_new_tokens=8), b.generate(ids8, max_new_tokens=8)), B
    for g in f.stage.slots:
        del g.gemv_rows
    for g in b.stage.slots:
        g.gemv_rows = fp8_gemv_max_rows
    fa, ba, _ = _pair(cfg, max_batch=1, seed=99)
    assert torch.equal(f.generate(one, max_new_tokens=16, assistant_model=fa, num_assistant_tokens=3),
                       b.generate(one, max_new_tokens=16, assistant_model=ba, num_assistant_tokens=3))
    # DESIGN.md §2's criteria against the CPU oracle on the dequantized weights
    ids = synthetic_tokens(cfg, 1, 16)
    deq = {k: t.cpu() for k, t in deq.items()}
    with torch.no_grad():
        ref = O.OracleModel(cfg, deq, "sdpa_math").logits(ids)
        ref_e = O.OracleModel(cfg, deq, "eager").logits(ids)
    err, floor = O.rel_l2(f(ids).logits.cpu(), ref), O.rel_l2(ref_e, ref)
    assert err <= 1.25 * floor, (err, floor)


def test_full_width_7b_layer():
    """One Qwen2.5-7B-shaped decoder layer with the full lm_head, weights drawn and quantized on the device."""
    cfg = replace(C.QWEN25_7B, n_layers=1)
    f, b, _ = _pair(cfg, max_batch=8, max_seq=64, init="device")
    for B in (1, 3, 8):
        ids = synthetic_tokens(cfg, B, 16, seed=B)
        assert torch.equal(f(ids).logits, b(ids).logits), B
        assert torch.equal(f.generate(ids, max_new_tokens=6), b.generate(ids, max_new_tokens=6)), B


def test_save_load_round_trip(tmp_path):
    f = DistributedModel(C.TINY_QWEN3, training=False, max_batch=2, max_seq=64, quantization_config=QC)
    f.save_pretrained(str(tmp_path))
    g = DistributedModel(str(tmp_path), training=False, max_batch=2, max_seq=64)
    assert g.quantization is not None
    for a, c in ((f.stage.params.q8.view(torch.uint8), g.stage.params.q8.view(torch.uint8)),
                 (f.stage.params.scales, g.stage.params.scales), (f.stage.params.flat, g.stage.params.flat)):
        assert torch.equal(a, c)
    ids = synthetic_tokens(C.TINY_QWEN3, 2, 10)
    assert torch.equal(f.generate(ids, max_new_tokens=6), g.generate(ids, max_new_tokens=6))
    with pytest.raises(NotImplementedError):
        DistributedModel(str(tmp_path), max_batch=2, max_seq=64)          # training=True by default
    with pytest.raises(NotImplementedError):
        f.create_optimizer()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_stage_fp8_pipeline_equals_single_stage(tmp_path):
    import os
    import socket
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(root, "tests", "fp8_multigpu_worker.py"), str(tmp_path)]
    r = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=root), capture_output=True, text=True, timeout=600)
    errs = "".join(open(p).read() for p in sorted(map(str, tmp_path.glob("err*.txt"))))
    assert r.returncode == 0, errs or r.stderr[-4000:]
    r0, r1 = torch.load(tmp_path / "rank0.pt"), torch.load(tmp_path / "rank1.pt")
    assert r0["logits_equal"] and r0["gen_equal"]
    assert r0["gen_graph_vs_eager"] and r1["gen_graph_vs_eager"] and r0["gen_peer_vs_nccl"] and r1["gen_peer_vs_nccl"]
