"""2 and 4 GPUs: the score log of a pipeline (peer-ring and NCCL decode hops), greedy with logits processors and
sampled, equals the single-stage run bit for bit on every rank (skipped with fewer GPUs)."""
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


@pytest.mark.parametrize("world", [2, 4])
def test_scores_across_stages_equal_single_stage(tmp_path, world):
    """The log lives on the last stage and is broadcast from the last rank: every rank returns the same scores."""
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
           "127.0.0.1", "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "scores_multigpu_worker.py"),
           str(tmp_path)]
    r = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=600)
    errs = "".join(open(p).read() for p in sorted(map(str, tmp_path.glob("err*.txt"))))
    assert r.returncode == 0, errs or r.stderr[-4000:]
    for rank in range(world):
        res = torch.load(tmp_path / f"sc{rank}.pt")
        assert res["used_ring"], (rank, res)
        assert all(v for k, v in res.items()), (rank, res)
