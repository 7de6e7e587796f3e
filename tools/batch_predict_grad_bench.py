# -*- coding: utf-8 -*-
"""GP.batch_grad_predict against the per-vector loop (set_parameter_vector + grad_predict per posterior sample), the
step an integrated acquisition function takes at every iteration of its optimiser.

    python tools/batch_predict_grad_bench.py [--rounds 7] [--workload co2|matern52_3d]

One JSON line per (workload, n, ns, return_var, B):
  loop_ms_per_member          set_parameter_vector + grad_predict (dense solver on the device), host-clock median
  batch_ms_per_member         gp.batch_grad_predict, host-clock median
  speedup                     loop / batch
  equal                       the two routes' outputs are bit-identical (checked in the same run)
  card                        GPU name and power limit, read in the same run
Workloads: the CO2 GP of the hyper-parameter tutorial (a sum of four kernel products, fitted mean and white noise) at
n = 512 with B = 50, and Matern-5/2 3-D (the Bayesian-optimisation case) at n = 1024 with B = 32; ns = 1 (one
optimiser step at one point) and ns = 256, with and without return_var.  After a warm-up call of each route the two
alternate, one call each per round, and the medians over the rounds are reported.
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


def co2_gp(n, seed=0):
    k1 = 66 ** 2 * kernels.ExpSquaredKernel(metric=67 ** 2)
    k2 = 2.4 ** 2 * kernels.ExpSquaredKernel(90 ** 2) * kernels.ExpSine2Kernel(gamma=2 / 1.3 ** 2, log_period=0.0)
    k3 = 0.66 ** 2 * kernels.RationalQuadraticKernel(log_alpha=np.log(0.78), metric=1.2 ** 2)
    k4 = 0.18 ** 2 * kernels.ExpSquaredKernel(1.6 ** 2)
    rng = np.random.default_rng(seed)
    t = np.sort(rng.uniform(1958, 2003, n))
    y = 315 + 1.3 * (t - 1958) + 3 * np.sin(2 * np.pi * t) + 0.3 * rng.standard_normal(n)
    gp = george.GP(k1 + k2 + k3 + k4, mean=np.mean(y), fit_mean=True, white_noise=np.log(0.19 ** 2),
                   fit_white_noise=True)
    gp.compute(t)
    return gp, y, 1e-4, lambda ns: np.linspace(1950, 2010, ns)


def matern_gp(n, seed=0):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-3, 3, (n, 3))
    y = np.sin(x[:, 0]) * np.cos(x[:, 1]) + 0.1 * rng.standard_normal(n)
    gp = george.GP(1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3))
    gp.compute(x, 0.3)
    return gp, y, 0.05, lambda ns: np.random.default_rng(seed + 1).uniform(-3, 3, (ns, 3))


def loop(gp, vecs, y, t, rv):
    p0 = gp.get_parameter_vector()
    res = []
    for v in vecs:
        gp.set_parameter_vector(v)
        res.append(gp.grad_predict(y, t, return_var=rv))
    gp.set_parameter_vector(p0)
    return tuple(np.stack([r[k] for r in res]) for k in range(len(res[0])))


def batch(gp, vecs, y, t, rv):
    return gp.batch_grad_predict(vecs, y, t, return_var=rv)


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--workload", default=None, help="run only this workload")
    args = ap.parse_args()
    gpu = card()
    work = [("co2", co2_gp, 512, 50), ("matern52_3d", matern_gp, 1024, 32)]
    for name, make, n, nb in work:
        if args.workload not in (None, name):
            continue
        gp, y, scale, points = make(n)
        gp.log_likelihood(y)
        rng = np.random.default_rng(n)
        vecs = gp.get_parameter_vector() + scale * rng.standard_normal((nb, len(gp)))
        for ns in (1, 256):
            t = points(ns)
            for rv in (False, True):
                want = loop(gp, vecs, y, t, rv)  # warm-up of this shape (workspace, code paths) for both routes
                got = batch(gp, vecs, y, t, rv)
                equal = all(np.array_equal(a, b) for a, b in zip(got, want))
                t_loop, t_batch = [], []
                for _ in range(args.rounds):  # alternate the two routes
                    dt, out = timed(lambda: loop(gp, vecs, y, t, rv))
                    t_loop.append(dt)
                    equal = equal and all(np.array_equal(a, b) for a, b in zip(out, want))
                    dt, out = timed(lambda: batch(gp, vecs, y, t, rv))
                    t_batch.append(dt)
                    equal = equal and all(np.array_equal(a, b) for a, b in zip(out, want))
                ml, mb = float(np.median(t_loop)), float(np.median(t_batch))
                print(json.dumps({
                    "workload": name, "n": n, "ns": ns, "return_var": rv, "B": nb,
                    "loop_ms_per_member": round(ml * 1e3 / nb, 4),
                    "batch_ms_per_member": round(mb * 1e3 / nb, 4),
                    "speedup": round(ml / mb, 2),
                    "equal": bool(equal),
                    "card": gpu}), flush=True)


if __name__ == "__main__":
    main()
