# -*- coding: utf-8 -*-
"""GP.batch_sample_conditional(rng=g) against the per-vector loop (set_parameter_vector + sample_conditional(rng=g)
per chain sample), the last step after an MCMC run: posterior predictive draws for every sample of a chain.

    python tools/batch_sample_bench.py [--reps 5] [--workload co2|matern52_3d]

One JSON line per (workload, n, ns, size, B):
  loop_ms / batch_ms            median host-clock time of one call (both return host arrays, so each ends in a
                                device synchronisation)
  loop_spread / batch_spread    (min, max) over the repetitions
  speedup                       loop_ms / batch_ms
  bit_equal                     the batch equals the loop bit for bit, and the generators end in the same state
  card                          GPU name and power limit, read in the same run
Workloads: the CO2 GP of the hyper-parameter tutorial (a sum of four kernel products, fitted mean and white noise) at
n = 512 with B = 50 members, ns in {256, 1024} and size in {1, 16, 256}, which covers both product paths and draws
costing from much less to about as much as the covariance; Matern-5/2 3-D at n = 4096, where the factorisation
dominates.  Each shape is warmed up once; the loop and the batch then alternate --reps times in the same process.
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
    # jitter: well above the rounding of a covariance whose prior variance is 66^2, far below the noise 0.19^2
    return gp, y, 1e-4, 1e-3, lambda ns: np.linspace(1950, 2010, ns)


def matern_gp(n, seed=0):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-3, 3, (n, 3))
    y = np.sin(x[:, 0]) * np.cos(x[:, 1]) + 0.1 * rng.standard_normal(n)
    gp = george.GP(1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3))
    gp.compute(x, 0.3)
    return gp, y, 0.05, 1e-6, lambda ns: np.random.default_rng(seed + 1).uniform(-3, 3, (ns, 3))


def loop(gp, vecs, y, t, size, rng, jitter):
    p0 = gp.get_parameter_vector()
    try:
        res = []
        for v in vecs:
            gp.set_parameter_vector(v)
            res.append(gp.sample_conditional(y, t, size, rng=rng, jitter=jitter))
    finally:
        gp.set_parameter_vector(p0)
    return np.stack(res)


def state(g):
    return json.dumps(g.bit_generator.state, sort_keys=True, default=str)


def run(name, make, n, nb, cases, reps, crd):
    gp, y, scale, jitter, points = make(n)
    gp.log_likelihood(y)
    vecs = gp.get_parameter_vector() + scale * np.random.default_rng(1).standard_normal((nb, len(gp)))
    for ns, size in cases:
        t = points(ns)
        calls = {
            "batch": lambda g: gp.batch_sample_conditional(vecs, y, t, size, rng=g, jitter=jitter),
            "loop": lambda g: loop(gp, vecs, y, t, size, g, jitter),
        }
        out, st = {}, {}
        for k, fn in calls.items():  # warm-up, and the outputs compared
            g = np.random.default_rng(7)
            out[k] = fn(g)
            st[k] = state(g)
        equal = bool(np.array_equal(out["batch"], out["loop"]) and st["batch"] == st["loop"])
        assert equal, (name, ns, size)
        times = {"batch": [], "loop": []}
        for _ in range(reps):
            for k in ("loop", "batch"):
                g = np.random.default_rng(7)
                t0 = time.perf_counter()
                calls[k](g)
                times[k].append(1e3 * (time.perf_counter() - t0))
        med = {k: float(np.median(v)) for k, v in times.items()}
        print(json.dumps({
            "workload": name, "n": n, "ns": ns, "size": size, "B": nb,
            "loop_ms": round(med["loop"], 2), "batch_ms": round(med["batch"], 2),
            "loop_spread": [round(min(times["loop"]), 2), round(max(times["loop"]), 2)],
            "batch_spread": [round(min(times["batch"]), 2), round(max(times["batch"]), 2)],
            "speedup": round(med["loop"] / med["batch"], 2), "bit_equal": equal, "card": crd,
        }), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--workload", choices=["co2", "matern52_3d"], default=None)
    a = ap.parse_args()
    assert george._lib.load().bgp_device_count() > 0, "no device: this benchmark measures the H100 path"
    crd = card()
    if a.workload in (None, "co2"):
        run("co2", co2_gp, 512, 50, [(ns, size) for ns in (256, 1024) for size in (1, 16, 256)], a.reps, crd)
    if a.workload in (None, "matern52_3d"):
        run("matern52_3d", matern_gp, 4096, 32, [(1000, 16)], a.reps, crd)


if __name__ == "__main__":
    main()
