# -*- coding: utf-8 -*-
"""GP.batch_grad_log_likelihood against the per-vector gradient loop (set_parameter_vector + grad_log_likelihood).

    python tools/batch_grad_bench.py [--min-seconds 1.0] [--workload co2|matern52_3d]

One JSON line per (workload, n, B):
  loop_ms_per_member          set_parameter_vector + grad_log_likelihood (dense solver on the device), wall time per
                              member
  batch_ms_per_member         gp.batch_grad_log_likelihood, wall time per member; split into
  batch_device_ms_per_member  one synchronised BasicSolver.batch_grad_terms timed with CUDA events, and
  batch_host_ms_per_member    the rest (host preparation of the members, the per-member composition)
  speedup                     loop / batch
  max_abs_diff                max |grad_batch - grad_loop| (0: bit-identical)
  card                        GPU name and power limit, read in the same run
Workloads (those of tools/batch_bench.py): the CO2 GP of the hyper-parameter tutorial (a sum of four kernel products,
fitted mean and white noise) at n = 512, B in {1, 8, 36, 64}; Matern-5/2 3-D at n in {1024, 4096}, B in {1, 32, 64}.
Every shape is warmed up first; the loop and the batch alternate, each timing repeating its call for at least
--min-seconds.
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
    return gp, y, 1e-4


def matern_gp(n, seed=0):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-3, 3, (n, 3))
    y = np.sin(x[:, 0]) * np.cos(x[:, 1]) + 0.1 * rng.standard_normal(n)
    gp = george.GP(1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3))
    gp.compute(x, 0.3)
    return gp, y, 0.05


def repeat(fn, min_seconds):
    """Mean wall seconds of fn() over at least min_seconds (and at least 3 calls)."""
    calls, t0 = 0, time.perf_counter()
    while True:
        fn()
        calls += 1
        el = time.perf_counter() - t0
        if calls >= 3 and el >= min_seconds:
            return el / calls


def loop(gp, vecs, y):
    p0 = gp.get_parameter_vector()
    out = np.empty((len(vecs), len(gp)))
    for b, v in enumerate(vecs):
        gp.set_parameter_vector(v)
        out[b] = gp.grad_log_likelihood(y)
    gp.set_parameter_vector(p0)
    return out


def device_ms(gp, vecs, y):
    """Milliseconds of one synchronised BasicSolver.batch_grad_terms on the members' host inputs, CUDA events around
    it."""
    import torch
    members = gp._batch_members(np.asarray(vecs, dtype=np.float64), y, gp._residual,
                                lambda y, c: y - (c + np.zeros(len(y))))
    spec, _, kpar, sigma, resid, _, _ = members
    which = gp.kernel.unfrozen_mask.astype(np.uint32)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    george.BasicSolver.batch_grad_terms(spec, kpar, gp._x, sigma, resid, which)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--workload", default=None, help="run only this workload")
    args = ap.parse_args()
    gpu = card()
    work = [("co2", co2_gp, 512, [1, 8, 36, 64]),
            ("matern52_3d", matern_gp, 1024, [1, 32, 64]),
            ("matern52_3d", matern_gp, 4096, [1, 32, 64])]
    for name, make, n, sizes in work:
        if args.workload not in (None, name):
            continue
        gp, y, scale = make(n)
        gp.log_likelihood(y)
        rng = np.random.default_rng(n)
        for nb in sizes:
            vecs = gp.get_parameter_vector() + scale * rng.standard_normal((nb, len(gp)))
            want = loop(gp, vecs, y)  # warm-up of this shape (workspace, code paths) for both routes
            got = gp.batch_grad_log_likelihood(vecs, y)
            diff = float(np.max(np.abs(got - want)))
            t_loop = t_batch = 0.0
            for _ in range(2):  # alternate the two routes
                t_loop += repeat(lambda: loop(gp, vecs, y), args.min_seconds) / 2
                t_batch += repeat(lambda: gp.batch_grad_log_likelihood(vecs, y), args.min_seconds) / 2
            dev = float(np.median([device_ms(gp, vecs, y) for _ in range(5)]))
            batch_ms = t_batch * 1e3 / nb
            print(json.dumps({
                "workload": name, "n": n, "B": nb,
                "loop_ms_per_member": round(t_loop * 1e3 / nb, 4),
                "batch_ms_per_member": round(batch_ms, 4),
                "batch_device_ms_per_member": round(dev / nb, 4),
                "batch_host_ms_per_member": round(max(batch_ms - dev / nb, 0.0), 4),
                "speedup": round(t_loop / t_batch, 2),
                "max_abs_diff": diff,
                "card": gpu}), flush=True)


if __name__ == "__main__":
    main()
