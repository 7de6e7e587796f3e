# -*- coding: utf-8 -*-
"""GP.predict's variance / covariance: the reference's host route (``GP._predict_host``: K(x*, x) downloaded,
``solver.apply_inverse`` on its transpose, numpy reduction) against the device path (``solver.predictive``), in one
process and alternating the two.

    python tools/predict_bench.py [--reps 3] [--out DIR]

Workloads (the sizes DESIGN.md §6 quotes):
  HODLR  Matern-3/2, N = 2^18, leaf 256, tol 1e-10, exhaust="lowrank": variance at ns = 256, 1024, 4096, covariance at
         ns = 1024;
  dense  Matern-5/2 3-D, N = 32768: variance and covariance at ns = 1024.
Each line reports the wall time of both paths (median over --reps; every call ends in a device synchronise), the
device time of each phase of one device call (torch.profiler, in a separate profiled call: kernel-matrix build,
solve, reduction / GEMM, copies) and the largest difference between the two outputs on the prior's scale.  The host
path at ns = 4096 holds three (N, ns) float64 arrays (~26 GB); where the host has less memory available it is reported
as skipped.
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
from george_b200 import kernels  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, universal_newlines=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception:
        return "unknown"


def mem_available():
    try:
        with open("/proc/meminfo") as fh:
            for line in fh:
                if line.startswith("MemAvailable:"):
                    return int(line.split()[1]) * 1024
    except OSError:
        pass
    return 0


def phase_of(name):
    if "predict_var" in name or "gemm_dmma" in name or "predict_slices" in name:
        return "reduce_ms"
    if "kmat_" in name:
        return "build_ms"
    return "solve_ms"


def device_phases(fn):
    """Device time per phase of one call of ``fn``, from torch.profiler's CUDA activity records."""
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
        for _ in range(2):  # the first session starts the activity tracer and can miss the first kernels: discard it
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
        out = {"build_ms": 0.0, "solve_ms": 0.0, "reduce_ms": 0.0, "copy_ms": 0.0, "build_kernels": []}
        for e in prof.events():
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = e.cuda_time_total
            if t <= 0:
                continue
            key = "copy_ms" if e.name.lower().startswith("memcpy") or e.name.lower().startswith("memset") else phase_of(e.name)
            out[key] += t * 1e-3
            if key == "build_ms" and e.name[:60] not in out["build_kernels"]:
                out["build_kernels"].append(e.name[:60])
        return out
    except Exception as exc:  # the measurement needs torch with CUDA; never fall back to another clock
        return {"phases": "not measured ({0})".format(type(exc).__name__)}


def wall(fn):
    t0 = time.perf_counter()
    r = fn()
    return (time.perf_counter() - t0) * 1e3, r


def run_case(label, gp, y, t, what, reps, host_ok):
    xs = gp.parse_samples(t)
    alpha = gp._compute_alpha(y, True)
    dev = lambda: gp.solver.predictive(gp.kernel, xs, what)  # noqa: E731
    host = lambda: gp._predict_host(alpha, xs, what == "var", gp.kernel)[1]  # noqa: E731
    dev()  # warm-up (module load, pool allocation)
    if host_ok:
        host()
    td, th = [], []
    out_d = out_h = None
    for _ in range(reps):
        if host_ok:
            ms, out_h = wall(host)
            th.append(ms)
        ms, out_d = wall(dev)
        td.append(ms)
    scale = np.max(np.abs(gp.kernel.get_value(xs[:256], diag=True)))
    rec = {"case": label, "what": what, "ns": int(xs.shape[0]), "device_ms": float(np.median(td)),
           "host_ms": float(np.median(th)) if host_ok else "host path skipped",
           "max_diff_over_prior": float(np.max(np.abs(out_d - out_h)) / scale) if host_ok else "not measured"}
    rec.update(device_phases(dev))
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for predict_bench.json")
    a = ap.parse_args()
    info = {"card": card(), "host_mem_available_gb": mem_available() / 2 ** 30}
    print(json.dumps(info))
    records = []
    rng = np.random.default_rng(7)

    n = 1 << 18
    x = np.sort(rng.uniform(0, 2000, n))
    y = np.sin(x) + 0.1 * rng.normal(size=n)
    gp = george.GP(1.0 * kernels.Matern32Kernel(4.0), solver=george.HODLRSolver, min_size=256, tol=1e-10,
                   exhaust="lowrank")
    gp.compute(x, 0.1)
    for ns, what in ((256, "var"), (1024, "var"), (4096, "var"), (1024, "cov")):
        need = 3.2 * 8.0 * n * ns
        t = rng.uniform(-5, 2005, ns)
        rec = run_case("hodlr_m32_n262144", gp, y, t, what, a.reps, mem_available() > need)
        print(json.dumps(rec))
        records.append(rec)
    del gp

    n = 32768
    x = rng.uniform(0, 1, (n, 3))
    x = x[np.argsort(x[:, 0])]
    y = np.sin(x.sum(axis=1))
    gp = george.GP(1.0 * kernels.Matern52Kernel(0.5, ndim=3))
    gp.compute(x, 0.1)
    t = rng.uniform(0, 1, (1024, 3))
    for what in ("var", "cov"):
        rec = run_case("dense_m52_3d_n32768", gp, y, t, what, a.reps, True)
        print(json.dumps(rec))
        records.append(rec)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "predict_bench.json"), "w") as fh:
            json.dump(dict(info, records=records), fh, indent=1)


if __name__ == "__main__":
    main()
