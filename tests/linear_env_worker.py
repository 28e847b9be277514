"""Runs the exact and rounding legs of tests/linear_cases.py for the GEMV and GEMM kernels in a fresh process, so that
the settings the library reads once (TL_GEMV_IMPL, TL_GEMV_CTAS_PER_SM, TL_GEMV_RING_KB, TL_PDL) take effect.

    python tests/linear_env_worker.py OUT.json

writes {"errors": [...], "path_error": "...", "bits": {case/leg: sha-256 of C}, "ratios": {...}}."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from tests import linear_cases as L  # noqa: E402

GEMM_NAMES = ("gemm.kk.bias_res.t32", "gemm.kB.acc_bf16.t128", "gemm.split4", "gemm.norm.fused", "gemm.AB.k52.acc")
GEMV_FORMS = ("bias", "res_inplace", "swiglu", "norm_swiglu")


def cases(sms):
    gemv = [c for c in L.gemv_path_matrix(sms)
            if c.name.startswith("gemv.fallback") or (c.M in (1, 3, 5, 8) and c.name.split(".")[2] in GEMV_FORMS)]
    gemm = [c for c in L.gemm_path_matrix(sms) if c.name in GEMM_NAMES]
    return gemv + L.gemv_reg_cases(sms) + gemm


def main(out_path):
    from tensorlink_b200 import native as nat
    nat.require_device()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    launch = L.native_launch(nat)
    res = {"errors": [], "bits": {}, "ratios": {}, "sms": sms}
    expected = []
    with L.KernelLog() as log:
        for c in cases(sms):
            for leg in ("exact", "round"):
                if leg == "exact" and not c.exact_ok:
                    continue
                r = L.check_call(c, leg, launch, "cuda", sms, want_bits=True)
                res["errors"] += r["errors"]
                res["bits"][f"{c.name}/{leg}"] = r["bits_c"]
                fam = c.op + (".norm" if c.norm else "")
                res["ratios"][fam] = max(res["ratios"].get(fam, 0.0), r["ratio"])
                expected.append((f"{c.name}/{leg}", r["path"]["kernels"]))
    res["path_error"] = L.match_paths(expected, log.kernels, log.all_names)
    res["n_kernels"] = len(log.kernels)
    with open(out_path, "w") as f:
        json.dump(res, f)


if __name__ == "__main__":
    main(sys.argv[1])
