# -*- coding: utf-8 -*-
"""The GP.batch_* methods against the per-vector loops they replace (set_parameter_vector, then the one-vector method).

    python tools/batch_bench.py --entry {log_likelihood,grad,predict,grad_predict,sample,loo,fisher}
        [--workload co2|matern52_3d|matern32_1d]
        [--min-seconds 1.0] [--cpu-members 4] [--kind mean|var|cov] [--rounds 7] [--reps 5]

One JSON line per shape.  Every line has
  batch_device_ms_per_member  the BasicSolver.batch_* hook the GP calls, timed with CUDA events around one
                              synchronised call (median of 5 calls of the public method)
  card                        GPU name and power limit, read in the same run
and the fields of its entry:
  log_likelihood  GP.batch_log_likelihood(quiet=True) against log_likelihood: loop_ms_per_member and
                  batch_ms_per_member (wall time per member), batch_host_ms_per_member (batch minus device), speedup
                  (loop / batch), cpu_ms_per_member (the CPU route of bench.py's dense_secondary: oracle.value_symmetric
                  + scipy cholesky / cho_solve, LAPACK on cpu_threads threads, on --cpu-members members), max_rel_diff
                  (max |ll_batch - ll_loop| / max(1, |ll_loop|)), nonfinite_members
  grad            GP.batch_grad_log_likelihood against grad_log_likelihood: the timings of log_likelihood and
                  max_abs_diff (0: bit-identical)
  predict         GP.batch_predict against predict, per --kind: the timings of grad and max_abs_diff over the mean and
                  var / cov
  grad_predict    GP.batch_grad_predict against grad_predict, with and without return_var: loop_ms_per_member and
                  batch_ms_per_member (host-clock medians over --rounds alternating rounds), speedup and equal (the
                  outputs are bit-identical in every round)
  sample          GP.batch_sample_conditional(rng=g) against sample_conditional(rng=g): loop_ms / batch_ms (median
                  host-clock time of one call over --reps alternating repetitions), loop_spread / batch_spread (min,
                  max), speedup and bit_equal (the draws and the generators' final states are equal)
  loo             GP.batch_loo_predict, batch_loo_log_likelihood(quiet=True) and
                  batch_grad_loo_log_likelihood(quiet=True, return_value=True) against loo_predict,
                  loo_log_likelihood and grad_loo_log_likelihood, per method: loop_ms_per_member and
                  batch_ms_per_member (host-clock medians over --rounds alternating rounds), loop_spread / batch_spread
                  (min, max per member), speedup and equal (the outputs are bit-identical in every round)
  fisher          GP.batch_fisher_information(quiet=True), without and with y, against fisher_information: the fields
                  of loo
Workloads: the CO2 GP of the hyper-parameter tutorial (a sum of four kernel products, fitted mean and white noise),
Matern-5/2 3-D (the Bayesian-optimisation case) and Matern-3/2 1-D (a light curve with a fitted mean and white noise,
the Fisher information's large case), at the sizes listed in each entry's table below: the sizes a sampler's step, a
posterior-predictive pass or an acquisition optimiser's step uses.  Every shape is warmed up first, through
both routes.
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
    """``(gp, y, scale, points)``: the computed GP, its data, the spread of the members around its parameter vector
    and ``points(ns)``, the test points."""
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
    """As :func:`co2_gp`."""
    rng = np.random.default_rng(seed)
    x = rng.uniform(-3, 3, (n, 3))
    y = np.sin(x[:, 0]) * np.cos(x[:, 1]) + 0.1 * rng.standard_normal(n)
    gp = george.GP(1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3))
    gp.compute(x, 0.3)
    return gp, y, 0.05, lambda ns: np.random.default_rng(seed + 1).uniform(-3, 3, (ns, 3))


def matern32_gp(n, seed=0):
    """As :func:`co2_gp`."""
    rng = np.random.default_rng(seed)
    t = np.sort(rng.uniform(0, 100, n))
    y = np.sin(t / 3) + 0.1 * rng.standard_normal(n)
    gp = george.GP(1.3 * kernels.Matern32Kernel(4.0), mean=0.1, fit_mean=True, white_noise=np.log(0.05),
                   fit_white_noise=True)
    gp.compute(t, 0.3)
    return gp, y, 0.05, lambda ns: np.linspace(0, 100, ns)


MODELS = {"co2": co2_gp, "matern52_3d": matern_gp, "matern32_1d": matern32_gp}


def repeat(fn, min_seconds):
    """Mean wall seconds of fn() over at least min_seconds (and at least 3 calls)."""
    calls, t0 = 0, time.perf_counter()
    while True:
        fn()
        calls += 1
        el = time.perf_counter() - t0
        if calls >= 3 and el >= min_seconds:
            return el / calls


def timed(fn):
    """(wall seconds, result) of one call of fn."""
    t0 = time.perf_counter()
    out = fn()
    return time.perf_counter() - t0, out


def loop(gp, vecs, fn):
    """[fn() for each member] with the member's parameter vector set, the GP's restored after."""
    p0 = gp.get_parameter_vector()
    try:
        res = []
        for v in vecs:
            gp.set_parameter_vector(v)
            res.append(fn())
    finally:
        gp.set_parameter_vector(p0)
    return res


class TimedSolver(george.BasicSolver):
    """BasicSolver whose batch_* hooks record the device time of each call in ``ms``."""
    ms = []


def _timed_hook(name):
    base = getattr(george.BasicSolver, name)

    def hook(*args):
        import torch
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = base(*args)
        e1.record()
        torch.cuda.synchronize()
        TimedSolver.ms.append(e0.elapsed_time(e1))
        return out
    return staticmethod(hook)


for _name in ("batch_log_likelihood", "batch_grad_terms", "batch_predict", "batch_predict_grad", "batch_sample",
              "batch_loo_terms", "batch_fisher_terms"):
    setattr(TimedSolver, _name, _timed_hook(_name))


def device_ms(gp, call, calls=5):
    """Median milliseconds of the solver hook inside ``call()`` (a GP.batch_* call on ``gp``)."""
    saved, gp.solver_type, TimedSolver.ms = gp.solver_type, TimedSolver, []
    try:
        for _ in range(calls):
            call()
    finally:
        gp.solver_type = saved
    return float(np.median(TimedSolver.ms))


def vectors(gp, scale, nb, rng):
    return gp.get_parameter_vector() + scale * rng.standard_normal((nb, len(gp)))


def cpu_route(gp, vecs, y, members):
    import oracle
    import scipy.linalg
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


def per_member(t_loop, t_batch, dev, nb):
    """The wall-time fields of the log_likelihood, grad and predict entries."""
    batch_ms = t_batch * 1e3 / nb
    return {"loop_ms_per_member": round(t_loop * 1e3 / nb, 4), "batch_ms_per_member": round(batch_ms, 4),
            "batch_device_ms_per_member": round(dev / nb, 4),
            "batch_host_ms_per_member": round(max(batch_ms - dev / nb, 0.0), 4),
            "speedup": round(t_loop / t_batch, 2)}


def alternate(loop_fn, batch_fn, min_seconds):
    """Mean wall seconds of the loop and the batch, alternating the two routes."""
    t_loop = t_batch = 0.0
    for _ in range(2):
        t_loop += repeat(loop_fn, min_seconds) / 2
        t_batch += repeat(batch_fn, min_seconds) / 2
    return t_loop, t_batch


def bench_log_likelihood(args, emit):
    """CO2 at n = 512 with B in {1, 8, 36, 64}; Matern-5/2 3-D at n in {1024, 4096} with B in {1, 32, 64}."""
    work = [("co2", 512, [1, 8, 36, 64]), ("matern52_3d", 1024, [1, 32, 64]), ("matern52_3d", 4096, [1, 32, 64])]
    for name, n, sizes in work:
        if args.workload not in (None, name):
            continue
        gp, y, scale, _ = MODELS[name](n)
        gp.log_likelihood(y)
        rng = np.random.default_rng(n)
        cpu_ms = None
        for nb in sizes:
            vecs = vectors(gp, scale, nb, rng)
            batch = lambda: gp.batch_log_likelihood(vecs, y, quiet=True)  # noqa: E731
            one = lambda: np.array(loop(gp, vecs, lambda: gp.log_likelihood(y, quiet=True)))  # noqa: E731
            batch()  # warm-up of this shape (workspace, code paths)
            ll_loop, ll_batch = one(), batch()
            t_loop, t_batch = repeat(one, args.min_seconds), repeat(batch, args.min_seconds)
            dev = device_ms(gp, batch)
            if cpu_ms is None:
                cpu_ms = cpu_route(gp, vecs if nb >= args.cpu_members else
                                   vectors(gp, scale, args.cpu_members, rng), y, args.cpu_members)
            fin = np.isfinite(ll_loop)
            diff = float(np.max(np.abs(ll_batch[fin] - ll_loop[fin]) / np.maximum(1.0, np.abs(ll_loop[fin])))) \
                if fin.any() else None
            emit(dict({"workload": name, "n": n, "B": nb}, **per_member(t_loop, t_batch, dev, nb),
                      cpu_ms_per_member=round(cpu_ms, 3), cpu_threads=cpu_threads(), max_rel_diff=diff,
                      nonfinite_members=int((~fin).sum())))


def bench_grad(args, emit):
    """The workloads of bench_log_likelihood."""
    work = [("co2", 512, [1, 8, 36, 64]), ("matern52_3d", 1024, [1, 32, 64]), ("matern52_3d", 4096, [1, 32, 64])]
    for name, n, sizes in work:
        if args.workload not in (None, name):
            continue
        gp, y, scale, _ = MODELS[name](n)
        gp.log_likelihood(y)
        rng = np.random.default_rng(n)
        for nb in sizes:
            vecs = vectors(gp, scale, nb, rng)
            batch = lambda: gp.batch_grad_log_likelihood(vecs, y)  # noqa: E731
            one = lambda: np.stack(loop(gp, vecs, lambda: gp.grad_log_likelihood(y)))  # noqa: E731
            want = one()  # warm-up of this shape (workspace, code paths) for both routes
            diff = float(np.max(np.abs(batch() - want)))
            t_loop, t_batch = alternate(one, batch, args.min_seconds)
            emit(dict({"workload": name, "n": n, "B": nb}, **per_member(t_loop, t_batch, device_ms(gp, batch), nb),
                      max_abs_diff=diff))


def bench_predict(args, emit):
    """CO2 at n = 512, ns = 250, B in {1, 8, 50}, for mean, var and cov; Matern-5/2 3-D at n in {1024, 4096},
    ns = 1000, B in {1, 32}, for var and cov."""
    work = [("co2", 512, 250, ["mean", "var", "cov"], [1, 8, 50]),
            ("matern52_3d", 1024, 1000, ["var", "cov"], [1, 32]),
            ("matern52_3d", 4096, 1000, ["var", "cov"], [1, 32])]
    kwargs_of = {"mean": dict(return_cov=False), "var": dict(return_var=True), "cov": dict(return_cov=True)}
    for name, n, ns, kinds, sizes in work:
        if args.workload not in (None, name):
            continue
        gp, y, scale, points = MODELS[name](n)
        t = points(ns)
        gp.log_likelihood(y)
        rng = np.random.default_rng(n)
        for kind in [k for k in kinds if args.kind in (None, k)]:
            kw = kwargs_of[kind]
            for nb in sizes:
                vecs = vectors(gp, scale, nb, rng)
                batch = lambda: gp.batch_predict(vecs, y, t, **kw)  # noqa: E731
                one = lambda: loop(gp, vecs, lambda: gp.predict(y, t, **kw))  # noqa: E731
                want = one()  # warm-up of this shape (workspace, code paths) for both routes
                want = (np.stack(want),) if kind == "mean" else tuple(np.stack([r[k] for r in want]) for k in (0, 1))
                got = batch()
                got = got if isinstance(got, tuple) else (got,)
                diff = max(float(np.max(np.abs(a - b))) if a.size else 0.0 for a, b in zip(got, want))
                t_loop, t_batch = alternate(one, batch, args.min_seconds)
                emit(dict({"workload": name, "n": n, "ns": ns, "kind": kind, "B": nb},
                          **per_member(t_loop, t_batch, device_ms(gp, batch), nb), max_abs_diff=diff))


def bench_grad_predict(args, emit):
    """CO2 at n = 512 with B = 50 and Matern-5/2 3-D at n = 1024 with B = 32; ns = 1 (one optimiser step at one
    point) and ns = 256, with and without return_var."""
    for name, n, nb in [("co2", 512, 50), ("matern52_3d", 1024, 32)]:
        if args.workload not in (None, name):
            continue
        gp, y, scale, points = MODELS[name](n)
        gp.log_likelihood(y)
        vecs = vectors(gp, scale, nb, np.random.default_rng(n))
        for ns in (1, 256):
            t = points(ns)
            for rv in (False, True):
                def one():
                    res = loop(gp, vecs, lambda: gp.grad_predict(y, t, return_var=rv))
                    return tuple(np.stack([r[k] for r in res]) for k in range(len(res[0])))
                batch = lambda: gp.batch_grad_predict(vecs, y, t, return_var=rv)  # noqa: E731
                want = one()  # warm-up of this shape (workspace, code paths) for both routes
                equal = all(np.array_equal(a, b) for a, b in zip(batch(), want))
                t_loop, t_batch = [], []
                for _ in range(args.rounds):  # alternate the two routes
                    for fn, ts in ((one, t_loop), (batch, t_batch)):
                        dt, out = timed(fn)
                        ts.append(dt)
                        equal = equal and all(np.array_equal(a, b) for a, b in zip(out, want))
                ml, mb = float(np.median(t_loop)), float(np.median(t_batch))
                emit({"workload": name, "n": n, "ns": ns, "return_var": rv, "B": nb,
                      "loop_ms_per_member": round(ml * 1e3 / nb, 4), "batch_ms_per_member": round(mb * 1e3 / nb, 4),
                      "batch_device_ms_per_member": round(device_ms(gp, batch) / nb, 4),
                      "speedup": round(ml / mb, 2), "equal": bool(equal)})


def bench_sample(args, emit):
    """CO2 at n = 512 with B = 50, ns in {256, 1024} and size in {1, 16, 256}, which covers both product paths and
    draws costing from much less to about as much as the covariance; Matern-5/2 3-D at n = 4096, where the
    factorisation dominates."""
    # jitter: for CO2 well above the rounding of a covariance whose prior variance is 66^2, far below the noise 0.19^2
    work = [("co2", 512, 50, 1e-3, [(ns, size) for ns in (256, 1024) for size in (1, 16, 256)]),
            ("matern52_3d", 4096, 32, 1e-6, [(1000, 16)])]
    state = lambda g: json.dumps(g.bit_generator.state, sort_keys=True, default=str)  # noqa: E731
    for name, n, nb, jitter, cases in work:
        if args.workload not in (None, name):
            continue
        gp, y, scale, points = MODELS[name](n)
        gp.log_likelihood(y)
        vecs = vectors(gp, scale, nb, np.random.default_rng(1))
        for ns, size in cases:
            t = points(ns)
            calls = {
                "batch": lambda g: gp.batch_sample_conditional(vecs, y, t, size, rng=g, jitter=jitter),
                "loop": lambda g: np.stack(loop(gp, vecs, lambda: gp.sample_conditional(y, t, size, rng=g,
                                                                                         jitter=jitter))),
            }
            out, st = {}, {}
            for k, fn in calls.items():  # warm-up, and the outputs compared
                g = np.random.default_rng(7)
                out[k] = fn(g)
                st[k] = state(g)
            equal = bool(np.array_equal(out["batch"], out["loop"]) and st["batch"] == st["loop"])
            assert equal, (name, ns, size)
            times = {"batch": [], "loop": []}
            for _ in range(args.reps):
                for k in ("loop", "batch"):
                    times[k].append(1e3 * timed(lambda: calls[k](np.random.default_rng(7)))[0])
            med = {k: float(np.median(v)) for k, v in times.items()}
            dev = device_ms(gp, lambda: calls["batch"](np.random.default_rng(7)))
            emit({"workload": name, "n": n, "ns": ns, "size": size, "B": nb,
                  "loop_ms": round(med["loop"], 2), "batch_ms": round(med["batch"], 2),
                  "loop_spread": [round(min(times["loop"]), 2), round(max(times["loop"]), 2)],
                  "batch_spread": [round(min(times["batch"]), 2), round(max(times["batch"]), 2)],
                  "batch_device_ms_per_member": round(dev / nb, 4),
                  "speedup": round(med["loop"] / med["batch"], 2), "bit_equal": equal})


def bench_loo(args, emit):
    """CO2 at n = 512 with B in {8, 64}; Matern-5/2 3-D at n = 1024 and n = 4096 with B = 32."""
    methods = [
        ("predict", lambda gp, v, y: gp.batch_loo_predict(v, y), lambda gp, y: gp.loo_predict(y)),
        ("value", lambda gp, v, y: gp.batch_loo_log_likelihood(v, y, quiet=True),
         lambda gp, y: gp.loo_log_likelihood(y, quiet=True)),
        ("grad", lambda gp, v, y: gp.batch_grad_loo_log_likelihood(v, y, quiet=True, return_value=True),
         lambda gp, y: gp.grad_loo_log_likelihood(y, quiet=True, return_value=True)),
    ]
    work = [("co2", 512, [8, 64]), ("matern52_3d", 1024, [32]), ("matern52_3d", 4096, [32])]
    for name, n, sizes in work:
        if args.workload not in (None, name):
            continue
        gp, y, scale, _ = MODELS[name](n)
        gp.log_likelihood(y)
        rng = np.random.default_rng(n)
        for nb in sizes:
            vecs = vectors(gp, scale, nb, rng)
            for method, batch_fn, one_fn in methods:
                def one():
                    res = loop(gp, vecs, lambda: one_fn(gp, y))
                    if isinstance(res[0], tuple):
                        return tuple(np.stack([r[k] for r in res]) for k in range(len(res[0])))
                    return np.array(res)
                batch = lambda: batch_fn(gp, vecs, y)  # noqa: E731

                def same(a, b):
                    a, b = (a, b) if isinstance(a, tuple) else ((a,), (b,))
                    return all(np.array_equal(u, w) for u, w in zip(a, b))
                want = one()  # warm-up of this shape (workspace, code paths) for both routes
                equal = same(batch(), want)
                t_loop, t_batch = [], []
                for _ in range(args.rounds):  # alternate the two routes
                    for fn, ts in ((one, t_loop), (batch, t_batch)):
                        dt, out = timed(fn)
                        ts.append(dt * 1e3 / nb)
                        equal = equal and same(out, want)
                ml, mb = float(np.median(t_loop)), float(np.median(t_batch))
                emit({"workload": name, "n": n, "B": nb, "method": method,
                      "loop_ms_per_member": round(ml, 4), "batch_ms_per_member": round(mb, 4),
                      "loop_spread": [round(min(t_loop), 4), round(max(t_loop), 4)],
                      "batch_spread": [round(min(t_batch), 4), round(max(t_batch), 4)],
                      "batch_device_ms_per_member": round(device_ms(gp, batch) / nb, 4),
                      "speedup": round(ml / mb, 2), "equal": bool(equal)})


def bench_fisher(args, emit):
    """CO2 at n = 512 with B = 64, where a single call's rows are launch-bound; Matern-3/2 1-D at n = 4096 with
    B = 16, where they run near the tensor pipe's rate."""
    work = [("co2", 512, 64), ("matern32_1d", 4096, 16)]
    for name, n, nb in work:
        if args.workload not in (None, name):
            continue
        gp, y, scale, _ = MODELS[name](n)
        gp.log_likelihood(y)
        vecs = vectors(gp, scale, nb, np.random.default_rng(n))
        for method, yy in (("F", None), ("grad_F", y)):
            def one():
                res = loop(gp, vecs, lambda: gp.fisher_information(yy, quiet=True))
                if yy is None:
                    return np.stack(res)
                return np.stack([r[0] for r in res]), np.stack([r[1] for r in res])
            batch = lambda: gp.batch_fisher_information(vecs, yy, quiet=True)  # noqa: E731

            def same(a, b):
                a, b = (a, b) if isinstance(a, tuple) else ((a,), (b,))
                return all(np.array_equal(u, w) for u, w in zip(a, b))
            want = one()  # warm-up of this shape (workspace, code paths) for both routes
            equal = same(batch(), want)
            t_loop, t_batch = [], []
            for _ in range(args.rounds):  # alternate the two routes
                for fn, ts in ((one, t_loop), (batch, t_batch)):
                    dt, out = timed(fn)
                    ts.append(dt * 1e3 / nb)
                    equal = equal and same(out, want)
            ml, mb = float(np.median(t_loop)), float(np.median(t_batch))
            emit({"workload": name, "n": n, "B": nb, "method": method,
                  "loop_ms_per_member": round(ml, 4), "batch_ms_per_member": round(mb, 4),
                  "loop_spread": [round(min(t_loop), 4), round(max(t_loop), 4)],
                  "batch_spread": [round(min(t_batch), 4), round(max(t_batch), 4)],
                  "batch_device_ms_per_member": round(device_ms(gp, batch) / nb, 4),
                  "speedup": round(ml / mb, 2), "equal": bool(equal)})


ENTRIES = {"log_likelihood": bench_log_likelihood, "grad": bench_grad, "predict": bench_predict,
           "grad_predict": bench_grad_predict, "sample": bench_sample, "loo": bench_loo, "fisher": bench_fisher}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--entry", choices=sorted(ENTRIES), required=True)
    ap.add_argument("--workload", choices=sorted(MODELS), default=None, help="run only this workload")
    ap.add_argument("--min-seconds", type=float, default=1.0, help="log_likelihood, grad, predict: per timing")
    ap.add_argument("--cpu-members", type=int, default=4, help="log_likelihood: members of the CPU route")
    ap.add_argument("--kind", choices=["mean", "var", "cov"], default=None, help="predict: only this kind")
    ap.add_argument("--rounds", type=int, default=7, help="grad_predict, loo, fisher: alternating rounds")
    ap.add_argument("--reps", type=int, default=5, help="sample: alternating repetitions")
    args = ap.parse_args()
    assert george._lib.load().bgp_device_count() > 0, "no device: this benchmark measures the H100 path"
    gpu = card()
    ENTRIES[args.entry](args, lambda rec: print(json.dumps(dict(rec, card=gpu)), flush=True))


if __name__ == "__main__":
    main()
