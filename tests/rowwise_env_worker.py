"""Runs the AdamW cases of tests/rowwise_cases.py in a fresh process, so that TL_ADAM_STREAM (read once per process by
tl_adamw_step) takes effect.

    TL_ADAM_STREAM=0 python tests/rowwise_env_worker.py OUT.json

writes {"errors": [...], "ratio_p": ..., "ratio_mv": ..., "cases": n}."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests import rowwise_cases as R  # noqa: E402


def main(out_path):
    from tensorlink_b200 import native as nat
    nat.require_device()
    launch = R.NativeLaunch(nat)
    res = {"errors": [], "ratio_p": 0.0, "ratio_mv": 0.0, "cases": 0}
    runs = [dict(n=n, a=a, steps=R.ADAM_STEPS) for n in (7, 9, 4099, 2 ** 20 + 3) for a in R.ADAM_CFGS]
    spans, n_arena = R.stage_adam_spans([4096, 130, 70000], 4099)
    runs.append(dict(n=n_arena, a=R.ADAM_CFGS[3], steps=(1, 2, 10), spans=spans))
    runs.append(dict(n=4099, a=R.ADAM_CFGS[0], steps=(1, 10), zero_grad=True))
    for kw in runs:
        r = R.run_adam(kw.pop("n"), kw.pop("a"), kw.pop("steps"), launch, "cuda", **kw)
        res["errors"] += r["errors"]
        res["ratio_p"] = max(res["ratio_p"], r["ratio_p"])
        res["ratio_mv"] = max(res["ratio_mv"], r["ratio_mv"])
        res["cases"] += 1
    with open(out_path, "w") as f:
        json.dump(res, f)


if __name__ == "__main__":
    main(sys.argv[1])
