"""Short eager (no CUDA graph) generate for ncu: prefill + a few decode steps of the bench workload."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tensorlink_b200.ml import DistributedModel  # noqa: E402
from tensorlink_b200.ml.configs import get_config  # noqa: E402
from tensorlink_b200.ml.weights import synthetic_tokens  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--model", default="Qwen/Qwen2.5-7B")
ap.add_argument("--prompt", type=int, default=32)
ap.add_argument("--new", type=int, default=4)
ap.add_argument("--graph", action="store_true")
ap.add_argument("--rows", type=int, default=1, help="rows per decode step (32 = BASELINE config 5: wgmma GEMM + split-K path)")
ap.add_argument("--max-seq", type=int, default=0, help="KV cache length (> 2048 selects the split-KV decode attention)")
a = ap.parse_args()
cfg = get_config(a.model)
dm = DistributedModel(a.model, training=False, max_batch=a.rows, max_seq=a.max_seq or (a.prompt + a.new + 8), init="device",
                      max_tokens=a.rows * a.prompt)
ids = synthetic_tokens(cfg, a.rows, a.prompt).cuda()
torch.cuda.synchronize()
torch.cuda.cudart().cudaProfilerStart()
out = dm.generate(ids, max_new_tokens=a.new, use_graph=a.graph)
torch.cuda.synchronize()
torch.cuda.cudart().cudaProfilerStop()
print(out[0, -a.new:].tolist())
