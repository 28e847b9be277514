"""Timeline model of one pipelined training step (GPipe order, deferred weight gradients): which layer split is fastest?

Units: the forward of one decoder layer over one micro-batch = 1.  Per stage k with L_k layers (the last stage also
holds final norm + lm_head = HEAD layer-equivalents per GEMM):
  forward phase   F_k = L_k * f      (+ head forward; + head dgrad + head wgrad too when the head is NOT split)
  dgrad chain     B_k = L_k * b      (+ head dgrad when split)
  weight grads    W_k = n_mb * L_k * w (+ head) once, after the stage's last dgrad
Stages process micro-batches in order, a stage starts a micro-batch when the neighbour has delivered it.
Its unit costs are fixed inputs (tests/test_generate_host_cpu.py pins the step times they give); they have not been
re-measured on H100.

  python tools/pipeline_model.py --stages 8 --layers 28 --mb 16
"""
import argparse
import itertools


def step_time(split, n_mb, f=1.0, b=1.1, w=0.95, head=2.34, split_head=True, ms_per_unit=None):
    n = len(split)
    hf = head * (1.0 if split_head else 3.0)       # head work inside the forward phase
    hb = head if split_head else 0.0
    hw = head if split_head else 0.0
    F = [split[k] * f + (hf if k == n - 1 else 0.0) for k in range(n)]
    B = [split[k] * b + (hb if k == n - 1 else 0.0) for k in range(n)]
    W = [n_mb * (split[k] * w + (hw if k == n - 1 else 0.0)) for k in range(n)]
    # forward phase
    f_done = [[0.0] * n_mb for _ in range(n)]
    for k in range(n):
        t = 0.0
        for m in range(n_mb):
            ready = f_done[k - 1][m] if k else 0.0
            t = max(t, ready) + F[k]
            f_done[k][m] = t
    # dgrad chains (micro-batches in reverse), each stage after its own forward phase
    b_done = [[0.0] * n_mb for _ in range(n)]
    for k in reversed(range(n)):
        t = f_done[k][n_mb - 1]
        for i, m in enumerate(reversed(range(n_mb))):
            ready = b_done[k + 1][m] if k < n - 1 else 0.0
            t = max(t, ready) + B[k]
            b_done[k][m] = t
    end = [b_done[k][0] + W[k] for k in range(n)]
    return max(end), end


def best_split(n_stages, n_layers, n_mb, **kw):
    best = None
    lo, hi = max(0, n_layers // n_stages - 3), n_layers // n_stages + 3
    for head_layers in range(0, hi + 1):
        rest = n_layers - head_layers
        for combo in itertools.product(range(max(1, lo), hi + 1), repeat=n_stages - 1):
            if sum(combo) != rest:
                continue
            t, _ = step_time(list(combo) + [head_layers], n_mb, **kw)
            if best is None or t < best[0] - 1e-9:
                best = (t, list(combo) + [head_layers])
    return best


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--stages", type=int, default=8)
    ap.add_argument("--layers", type=int, default=28)
    ap.add_argument("--mb", type=int, default=None)
    ap.add_argument("--split", type=str, default=None, help="comma-separated layer counts to evaluate")
    a = ap.parse_args()
    n_mb = a.mb or 2 * a.stages
    ideal = n_mb * (a.layers * (1.0 + 1.1 + 0.95) + 3 * 2.34) / a.stages
    rows = []
    if a.split:
        sp = [int(x) for x in a.split.split(",")]
        for sh in (False, True):
            t, end = step_time(sp, n_mb, split_head=sh)
            rows.append((f"{sp} head {'split' if sh else 'fused in forward'}", t))
    t, sp = best_split(a.stages, a.layers, n_mb)
    rows.append((f"best split {sp} (head split)", t))
    for name, t in rows:
        print(f"{name}: {t:.1f} units, efficiency vs perfect balance {ideal / t:.3f}")
