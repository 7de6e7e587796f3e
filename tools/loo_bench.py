# -*- coding: utf-8 -*-
"""Time leave-one-out cross-validation against the marginal-likelihood gradient on the same handle.

    python tools/loo_bench.py [--reps 3] [--max-n 262144] [--dense-max-n 16384]

For each workload the GP is computed once, then ``GP.loo_log_likelihood`` (pass 1: alpha and d = diag(K^-1)),
``GP.grad_loo_log_likelihood`` (passes 1 and 2) and ``GP.grad_log_likelihood`` are each timed with a device
synchronise before and after, median of ``--reps`` after one warm-up call.  Workloads: ``BasicSolver`` at N = 4096 and
16384 (Matern-3/2 1-D) and bench.py's cfg3 on ``HODLRSolver`` (Matern-3/2 1-D, min_size=256, tol=1e-10,
exhaust="lowrank") at N = 2^16, 2^17 and 2^18.  Prints one JSON line per workload with the card's name and power limit,
read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import george_b200 as george  # noqa: E402
from george_b200 import _lib, kernels  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, universal_newlines=True, timeout=30)
    return r.stdout.strip().splitlines()[0]


def make_data(n):  # bench.py's inputs
    rng = np.random.default_rng(1234)
    x = np.sort(rng.uniform(0, 10 * n / 1000, n))
    yerr = 0.1 * np.ones(n)
    y = np.sin(x) + 0.1 * rng.normal(size=n)
    return x, yerr, y


def timed(fn, reps):
    lib = _lib.load()
    fn()  # warm-up: workspaces
    times = []
    for _ in range(reps):
        _lib.check(lib.bgp_dev_synchronize())
        t0 = time.perf_counter()
        fn()
        _lib.check(lib.bgp_dev_synchronize())
        times.append(time.perf_counter() - t0)
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--max-n", type=int, default=1 << 18)
    ap.add_argument("--dense-max-n", type=int, default=16384)
    args = ap.parse_args()
    os.environ.pop("BGP_GRAD_CHUNK", None)
    dev = card()
    cases = [("dense", n, george.BasicSolver, {}) for n in (4096, 16384) if n <= args.dense_max_n]
    cases += [("hodlr_cfg3", n, george.HODLRSolver, dict(min_size=256, tol=1e-10, seed=42, exhaust="lowrank"))
              for n in (1 << 16, 1 << 17, 1 << 18) if n <= args.max_n]
    for name, n, solver, kw in cases:
        x, yerr, y = make_data(n)
        gp = george.GP(1.0 * kernels.Matern32Kernel(1.0), solver=solver, **kw)
        gp.compute(x, yerr)
        reps = args.reps if n <= (1 << 17) else 1
        row = {"workload": name, "n": n, "card": dev,
               "loo_value_s": round(timed(lambda: gp.loo_log_likelihood(y), reps), 4),
               "loo_grad_s": round(timed(lambda: gp.grad_loo_log_likelihood(y, return_value=True), reps), 4),
               "ll_grad_s": round(timed(lambda: gp.grad_log_likelihood(y), reps), 4),
               "loo_value": gp.loo_log_likelihood(y), "log_likelihood": gp.log_likelihood(y)}
        row["loo_grad_over_ll_grad"] = round(row["loo_grad_s"] / row["ll_grad_s"], 3)
        print(json.dumps(row), flush=True)
        del gp


if __name__ == "__main__":
    main()
