"""N = 2 GPUs: a padded training step pipelined over two stages equals the single-stage step bit for bit (skipped with
fewer than 2 GPUs)."""
import os
import socket
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_padded_step_equals_single_stage(tmp_path):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "padded_multigpu_worker.py"), str(tmp_path)]
    r = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=600)
    errs = "".join(open(p).read() for p in sorted(map(str, tmp_path.glob("err*.txt"))))
    assert r.returncode == 0, errs or r.stderr[-4000:]
    ref = torch.load(tmp_path / "single.pt")
    for rank in (0, 1):
        got = torch.load(tmp_path / f"rank{rank}.pt")
        assert got["loss"] == ref["loss"]
        assert len(got["grads"]) > 5
        for k, v in got["grads"].items():
            assert torch.equal(v, ref["grads"][k]), f"rank {rank} grad {k} differs from the single-stage run"
