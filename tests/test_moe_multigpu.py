"""A two-stage Qwen3-MoE pipeline equals the single-stage run bit for bit (tests/moe_multigpu_worker.py)."""
import os
import socket
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_stage_moe_pipeline_equals_single_stage(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(root, "tests", "moe_multigpu_worker.py"), str(tmp_path)]
    r = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=root), capture_output=True, text=True, timeout=600)
    errs = "".join(open(p).read() for p in sorted(map(str, tmp_path.glob("err*.txt"))))
    assert r.returncode == 0, errs or r.stderr[-4000:]
    r0, r1 = torch.load(tmp_path / "rank0.pt"), torch.load(tmp_path / "rank1.pt")
    for B in (1, 8):
        assert r0[f"logits_equal_B{B}"] and r0[f"gen_equal_B{B}"], (B, r0)
        assert r0[f"gen_graph_vs_eager_B{B}"] and r1[f"gen_graph_vs_eager_B{B}"], (B, r0, r1)
