"""2 and 4 GPUs: generation with the logits processors through a pipeline (peer-ring and NCCL decode hops), greedy and
sampled, equals the single-stage run bit for bit (skipped with fewer GPUs)."""
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
def test_processors_across_stages_equal_single_stage(tmp_path, world):
    """The prompt reaches the last stage once, the history is kept there, the first token after prefill and every decode
    step append to it while the id goes into the first stage's mailbox (peer ring) or over NCCL."""
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
           "127.0.0.1", "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "logits_process_worker.py"),
           str(tmp_path)]
    r = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=600)
    errs = "".join(open(p).read() for p in sorted(map(str, tmp_path.glob("err*.txt"))))
    assert r.returncode == 0, errs or r.stderr[-4000:]
    for rank in range(world):
        res = torch.load(tmp_path / f"lp{rank}.pt")
        assert res["used_ring"] and res["sampled_differs"], (rank, res)
        for name in ("greedy", "sampled"):
            assert res[f"{name}_peer_vs_nccl"] and res[f"{name}_min_new_held"], (rank, name, res)
    r0 = torch.load(tmp_path / "lp0.pt")
    assert r0["greedy_vs_single"] and r0["sampled_vs_single"], r0
