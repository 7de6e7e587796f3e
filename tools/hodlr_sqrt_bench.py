# -*- coding: utf-8 -*-
"""Build and apply times of the HODLR symmetric factor K~ = W W^T (csrc/hodlr_sym.cu) at bench.py's workloads on one
GPU, beside the same factorisation's up-sweep time and a traffic bound for the apply.

    python tools/hodlr_sqrt_bench.py [--workloads cfg3,cfg2,cfg5] [--reps 3]

Build: the first symmetric_log_determinant after a compute(), device events around the build.  Apply:
apply_symmetric_factor on (N, size) standard normals, size 1, 8 and 64: the device time of the products (events, host
transfers excluded) and the host-clock time of the whole call (the host copies and pageable transfers included).
Bound: the factor panel P (N x sum r doubles) and the leaf factors read once per 64-column group, over 3.35 TB/s.
Prints one JSON line per workload.  Needs an H100."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

WORKLOADS = {"cfg3": (262144, 256), "cfg2": (65536, 100), "cfg5": (131072, 100)}


def kernel_of(name):
    from george_b200 import kernels as K
    if name == "cfg3":
        return 1.0 * K.Matern32Kernel(1.0)
    if name == "cfg2":
        return 1.0 * K.ExpSquaredKernel(1.0)
    return 1.0 * K.ExpSquaredKernel(1.0) + 0.5 * K.ExpSine2Kernel(gamma=1.0, log_period=np.log(3.0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg3,cfg2,cfg5")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    from george_b200.solvers._hodlr import HODLRSolver
    for name in args.workloads.split(","):
        n, min_size = WORKLOADS[name]
        x = np.sort(np.random.default_rng(1234).uniform(0, 10 * n / 1000, n))[:, None]
        s = HODLRSolver()
        builds, ups = [], []
        for _ in range(args.reps):
            s.compute(kernel_of(name), x, 0.1 * np.ones(n), min_size=min_size, tol=1e-10, seed=42, exhaust="lowrank")
            ups.append(s.timing()["upsweep_ms"])
            s.symmetric_log_determinant
            builds.append(s.symmetric_factor_timing()["build_ms"])
        w = s.work()
        leaf_bytes = 8.0 * w["leaf"] * n
        apply, apply_dev = {}, {}
        for size in (1, 8, 64):
            z = np.random.default_rng(0).standard_normal((n, size))
            s.apply_symmetric_factor(z)
            ts, td = [], []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                s.apply_symmetric_factor(z)
                ts.append(1e3 * (time.perf_counter() - t0))
                td.append(s.symmetric_factor_timing()["apply_ms"])
            apply[str(size)] = min(ts)
            apply_dev[str(size)] = min(td)
        bound_ms = 1e3 * (8.0 * n * w["R"] + leaf_bytes) / 3.35e12
        print(json.dumps({"workload": name, "N": n, "build_ms": min(builds), "upsweep_ms": min(ups),
                          "apply_device_ms": apply_dev, "apply_call_ms": apply, "apply_bound_ms_per_group": bound_ms, "R": w["R"]}))


if __name__ == "__main__":
    main()
