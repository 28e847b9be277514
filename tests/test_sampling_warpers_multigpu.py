"""2 GPUs: sampled generation with min_p / typical_p / epsilon_cutoff / eta_cutoff through a two-stage pipeline equals
the single-stage run bit for bit, and the sharp settings reproduce greedy decoding (skipped with fewer GPUs)."""
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


def test_warpers_across_two_stages(tmp_path):
    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
           "127.0.0.1", "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "warpers_multigpu_worker.py"),
           str(tmp_path)]
    r = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=600)
    errs = "".join(open(p).read() for p in sorted(map(str, tmp_path.glob("err*.txt"))))
    assert r.returncode == 0, errs or r.stderr[-4000:]
    for rank in range(world):
        res = torch.load(tmp_path / f"wp{rank}.pt")
        assert res["sharp_is_greedy"] and res["chain_differs"], (rank, res)
    r0 = torch.load(tmp_path / "wp0.pt")
    assert all(v for k, v in r0.items() if k.endswith("_vs_single") or k == "single_greedy_equal"), r0
