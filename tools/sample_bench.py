# -*- coding: utf-8 -*-
"""GP.sample_conditional with a caller's generator (the device route: predictive covariance, Cholesky and product on
the device) against the reference's host route (``predict`` + ``numpy.random.multivariate_normal``).

    python tools/sample_bench.py [--reps 3] [--out DIR] [--quick]

Workloads:
  dense  Matern-3/2 1-D, N = 4096 (BasicSolver);
  HODLR  Matern-3/2 1-D, N = 2^18, leaf 256, tol 1e-10, exhaust="lowrank" (bench.py's headline case);
  ns in {256, 1024, 4096, 8192} test points, size in {1, 16, 64, 256, 1024} draws.
Each line reports the device time of the three phases of one fused call (device events, bgp_sample_last_timing:
predictive covariance, symmetrisation + Cholesky, product), the wall time of the whole device call, and, at ns <= 1024
where it finishes in seconds, the wall time of the host route.  The product's two paths (a row kernel below
BGP_SAMPLE_DMMA_ROWS draws, the DMMA triangular GEMM from it) are compared directly on the dense factorisation
through bgp_mvn_sample at every size, which is what the threshold in include/bgp.h is chosen from.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import george_b200 as george  # noqa: E402
from george_b200 import _lib, kernels  # noqa: E402

NS = [256, 1024, 4096, 8192]
SIZES = [1, 16, 64, 256, 1024]
HOST_MAX_NS = 1024


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, universal_newlines=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception:
        return "unknown"


def phases():
    ms = (C.c_double * 3)()
    _lib.check(_lib.load().bgp_sample_last_timing(ms))
    return list(ms)


def make(solver, n, rng, **kw):
    t = np.sort(rng.uniform(0, n / 20.0, n))
    y = np.sin(t) + 0.1 * rng.standard_normal(n)
    gp = george.GP(1.0 * kernels.Matern32Kernel(1.0), solver=solver, **kw)
    gp.compute(t, 0.1)
    return gp, t, y


def median_time(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()  # every call ends in a device synchronise (or is host-only)
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def run_workload(label, gp, t, y, reps, ns_list, sizes, host):
    out = []
    lo, hi = t[0], t[-1]
    for ns in ns_list:
        ts = np.sort(np.random.default_rng(ns).uniform(lo, hi, ns))
        g = np.random.default_rng(7)
        gp.sample_conditional(y, ts, 1, rng=g)  # warm-up: alpha cached, modules loaded, this ns's workspace pooled
        for size in sizes:
            wall = median_time(lambda: gp.sample_conditional(y, ts, size, rng=g), reps)
            cov_ms, chol_ms, prod_ms = phases()
            rec = dict(workload=label, ns=ns, size=size, device_s=wall, cov_ms=cov_ms, chol_ms=chol_ms,
                       product_ms=prod_ms, product_path="rows" if size < _lib.BGP_SAMPLE_DMMA_ROWS else "dmma")
            if host and ns <= HOST_MAX_NS:
                np.random.seed(1)
                rec["host_s"] = median_time(lambda: gp.sample_conditional(y, ts, size), max(1, min(reps, 2)))
            print(json.dumps(rec), flush=True)
            out.append(rec)
    return out


def product_paths(gp, ns_list, sizes, reps):
    """The product alone, on one covariance through bgp_mvn_sample: each size runs on the path BGP_SAMPLE_DMMA_ROWS
    picks.  The row path's cost grows linearly with the draws and the DMMA path's is flat up to 128 draws (one tile
    column), so the crossover is the DMMA time at the threshold over the row path's time per draw."""
    out = []
    lib = _lib.load()
    for ns in ns_list:
        x = np.linspace(0, ns / 20.0, ns)[:, None]
        cov = gp.kernel.get_value(x)
        mean = np.zeros(ns)
        for size in sorted(set(sizes) | {_lib.BGP_SAMPLE_DMMA_ROWS - 1, _lib.BGP_SAMPLE_DMMA_ROWS, 2, 4, 8, 12}):
            if size < 1:
                continue
            z = np.random.default_rng(1).standard_normal((size, ns))
            o = np.empty((size, ns))
            ms = []
            for _ in range(reps + 1):
                _lib.check(lib.bgp_mvn_sample(_lib.ptr(cov), ns, _lib.ptr(mean), _lib.ptr(z), size, 1e-6, _lib.ptr(o)))
                ms.append(phases())
            ms = np.median(np.array(ms[1:]), axis=0)
            rec = dict(workload="product", ns=ns, size=size, chol_ms=ms[1], product_ms=ms[2],
                       product_ms_per_draw=ms[2] / size,
                       product_path="rows" if size < _lib.BGP_SAMPLE_DMMA_ROWS else "dmma")
            print(json.dumps(rec), flush=True)
            out.append(rec)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    ap.add_argument("--quick", action="store_true", help="ns = 256, 1024 and sizes 1, 64 only (a rehearsal)")
    args = ap.parse_args()
    ns_list, sizes = (NS[:2], [1, 64]) if args.quick else (NS, SIZES)
    head = dict(card=card(), threshold=_lib.BGP_SAMPLE_DMMA_ROWS)
    print(json.dumps(head), flush=True)
    rng = np.random.default_rng(0)
    recs = [head]
    gp, t, y = make(george.BasicSolver, 4096, rng)
    recs += product_paths(gp, ns_list, sizes, args.reps)
    recs += run_workload("dense N=4096", gp, t, y, args.reps, ns_list, sizes, host=True)
    del gp
    gp, t, y = make(george.HODLRSolver, 1 << 18, rng, min_size=256, tol=1e-10, exhaust="lowrank")
    recs += run_workload("hodlr N=262144", gp, t, y, args.reps, ns_list, sizes, host=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "sample_bench.json"), "w") as fh:
            json.dump(recs, fh, indent=1)


if __name__ == "__main__":
    main()
