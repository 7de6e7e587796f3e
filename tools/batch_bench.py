# -*- coding: utf-8 -*-
"""GP.batch_log_likelihood against the one-vector-at-a-time loop an ensemble sampler runs without it.

    python tools/batch_bench.py [--min-seconds 1.0] [--cpu-members 4]

One JSON line per (workload, n, B):
  loop_ms_per_member     set_parameter_vector + log_likelihood (dense solver on the device), wall time per member
  batch_ms_per_member    gp.batch_log_likelihood, wall time per member; split into
  batch_host_ms_per_member / batch_device_ms_per_member   host preparation, and the device call timed with CUDA events
                         around one synchronised BasicSolver.batch_log_likelihood
  speedup                loop / batch
  cpu_ms_per_member      the CPU route of bench.py's dense_secondary (oracle.value_symmetric + scipy cholesky /
                         cho_solve, LAPACK on cpu_threads threads), on --cpu-members members
  max_rel_diff           max |ll_batch - ll_loop| / max(1, |ll_loop|)
  card                   GPU name and power limit, read in the same run
Workloads: the CO2 GP of the hyper-parameter tutorial (a sum of four kernel products, fitted mean and white noise) at
n = 512 with B in {1, 8, 36, 64}; Matern-5/2 3-D at n in {1024, 4096} with B in {1, 32, 64}.  Every shape is warmed up
first and each timing repeats its call for at least --min-seconds.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.linalg

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import george_b200 as george  # noqa: E402
from george_b200 import kernels  # noqa: E402
from george_b200._spec import flatten  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, universal_newlines=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception:
        return "unknown"


def cpu_threads():
    try:
        from threadpoolctl import threadpool_info
        return max(i.get("num_threads", 0) for i in threadpool_info() if i.get("internal_api") != "openmp")
    except Exception:
        return os.cpu_count()


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
    out = np.empty(len(vecs))
    for b, v in enumerate(vecs):
        gp.set_parameter_vector(v)
        out[b] = gp.log_likelihood(y, quiet=True)
    gp.set_parameter_vector(p0)
    return out


def device_call(gp, vecs, y):
    """(device ms, host-argument ms) of one synchronised BasicSolver.batch_log_likelihood, timed with CUDA events."""
    import torch
    nb = len(vecs)
    t0 = time.perf_counter()
    full = np.tile(gp.get_parameter_vector(include_frozen=True), (nb, 1))
    full[:, gp.unfrozen_mask] = vecs
    nm, nw = gp.mean.full_size, gp.white_noise.full_size
    kpar = np.ascontiguousarray(full[:, nm + nw:])
    c = gp.white_noise.get_parameter_vector(include_frozen=True)
    sig = np.sqrt(gp._yerr2[None, :] + np.exp(full[:, nm:nm + 1] if type(gp.white_noise) is
                                              george.modeling.ConstantModel else c[0]))
    r = np.ascontiguousarray(np.broadcast_to(y, sig.shape) - (full[:, :1] if nm else 0.0))
    spec = flatten(gp.kernel)
    t1 = time.perf_counter()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    george.BasicSolver.batch_log_likelihood(spec, kpar, gp._x, sig, r)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), (t1 - t0) * 1e3


def cpu_route(gp, vecs, y, members):
    import oracle
    x = gp._x
    p0 = gp.get_parameter_vector()
    t0 = time.perf_counter()
    for v in vecs[:members]:
        gp.set_parameter_vector(v)
        K = oracle.value_symmetric(flatten(gp.kernel), x)
        K[np.diag_indices_from(K)] += gp._sigma(x) ** 2
        cf = scipy.linalg.cholesky(K, lower=False, overwrite_a=True)
        r = gp._residual_of(y)
        _ = -0.5 * (len(x) * np.log(2 * np.pi) + 2 * np.sum(np.log(np.diag(cf)))) \
            - 0.5 * r @ scipy.linalg.cho_solve((cf, False), r)
    gp.set_parameter_vector(p0)
    return (time.perf_counter() - t0) * 1e3 / min(members, len(vecs))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--cpu-members", type=int, default=4)
    args = ap.parse_args()
    gpu = card()
    work = [("co2", co2_gp, 512, [1, 8, 36, 64]), ("matern52_3d", matern_gp, 1024, [1, 32, 64]),
            ("matern52_3d", matern_gp, 4096, [1, 32, 64])]
    for name, make, n, sizes in work:
        gp, y, scale = make(n)
        gp.log_likelihood(y)
        rng = np.random.default_rng(n)
        cpu_ms = None
        for nb in sizes:
            vecs = gp.get_parameter_vector() + scale * rng.standard_normal((nb, len(gp)))
            gp.batch_log_likelihood(vecs, y, quiet=True)  # warm-up of this shape (workspace, code paths)
            ll_loop = loop(gp, vecs, y)
            ll_batch = gp.batch_log_likelihood(vecs, y, quiet=True)
            t_loop = repeat(lambda: loop(gp, vecs, y), args.min_seconds)
            t_batch = repeat(lambda: gp.batch_log_likelihood(vecs, y, quiet=True), args.min_seconds)
            dev = [device_call(gp, vecs, y) for _ in range(5)]
            dev_ms = float(np.median([d[0] for d in dev]))
            if cpu_ms is None:
                cpu_ms = cpu_route(gp, vecs if nb >= args.cpu_members else
                                   gp.get_parameter_vector() + scale * rng.standard_normal((args.cpu_members, len(gp))),
                                   y, args.cpu_members)
            fin = np.isfinite(ll_loop)
            diff = float(np.max(np.abs(ll_batch[fin] - ll_loop[fin]) / np.maximum(1.0, np.abs(ll_loop[fin])))) \
                if fin.any() else None
            batch_ms = t_batch * 1e3 / nb
            print(json.dumps({
                "workload": name, "n": n, "B": nb,
                "loop_ms_per_member": round(t_loop * 1e3 / nb, 4),
                "batch_ms_per_member": round(batch_ms, 4),
                "batch_device_ms_per_member": round(dev_ms / nb, 4),
                "batch_host_ms_per_member": round(max(batch_ms - dev_ms / nb, 0.0), 4),
                "speedup": round(t_loop / t_batch, 2),
                "cpu_ms_per_member": round(cpu_ms, 3), "cpu_threads": cpu_threads(),
                "max_rel_diff": diff, "nonfinite_members": int((~fin).sum()),
                "card": gpu}), flush=True)


if __name__ == "__main__":
    main()
