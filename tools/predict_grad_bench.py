# -*- coding: utf-8 -*-
"""GP.grad_predict(return_var=True) against GP.predict(return_var=True) and against the finite-difference loop a user
would otherwise run (2 * ndim + 1 calls of predict(return_var=True)), in one process, alternating the three.

    python tools/predict_grad_bench.py [--reps 5] [--out DIR]

Workloads (the sizes DESIGN.md §6 quotes):
  dense  Matern-5/2 3-D (axis-aligned metric), N = 1024 and 4096, ns = 1 (one optimiser step) and ns = 1024;
  HODLR  Matern-3/2 1-D, N = 2^18, leaf 256, tol 1e-10, exhaust="lowrank" (the headline model), ns = 4096.
Each line reports the wall time of the three (median over --reps; every call ends in a device synchronise) and the
card's name and power limit, read in the same run.
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


def fd_loop(gp, y, t, h=1e-5):
    """What a user runs without grad_predict: predict at t and at t +- h e_q for every axis q."""
    t2 = t.reshape(len(t), -1)
    out = [gp.predict(y, t, return_var=True)]
    for q in range(t2.shape[1]):
        for sgn in (1.0, -1.0):
            tq = t2.copy()
            tq[:, q] += sgn * h
            out.append(gp.predict(y, tq[:, 0] if t.ndim == 1 else tq, return_var=True))
    return out


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()  # every path copies its results to the host after a stream synchronise
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def run(name, gp, y, t, reps, name_card):
    calls = {
        "grad_predict_ms": lambda: gp.grad_predict(y, t, return_var=True),
        "predict_var_ms": lambda: gp.predict(y, t, return_var=True),
        "fd_loop_ms": lambda: fd_loop(gp, y, t),
    }
    for fn in calls.values():  # warm-up of every shape
        fn()
    ts = {k: [] for k in calls}
    for _ in range(reps):  # alternate the three
        for k, fn in calls.items():
            ts[k].append(timed(fn, 1))
    rec = dict(workload=name, ns=int(len(t)), card=name_card)
    rec.update({k: round(1e3 * float(np.median(v)), 3) for k, v in ts.items()})
    rec["grad_over_predict"] = round(rec["grad_predict_ms"] / rec["predict_var_ms"], 3)
    rec["fd_over_grad"] = round(rec["fd_loop_ms"] / rec["grad_predict_ms"], 3)
    print(json.dumps(rec), flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--skip-hodlr", action="store_true")
    a = ap.parse_args()
    name_card = card()
    print(json.dumps({"card": name_card}), flush=True)
    rng = np.random.default_rng(0)
    recs = []
    for n in (1024, 4096):
        x = rng.uniform(0, 10, (n, 3))
        y = np.sin(x[:, 0]) + np.cos(x[:, 1]) + 0.1 * rng.normal(size=n)
        gp = george.GP(kernels.Matern52Kernel([1.0, 2.0, 0.5], ndim=3))
        gp.compute(x, 0.1)
        for ns in (1, 1024):
            t = rng.uniform(0, 10, (ns, 3))
            recs.append(run("dense_m52_3d_n%d" % n, gp, y, t, a.reps, name_card))
    if not a.skip_hodlr:
        n = 1 << 18
        x = np.sort(rng.uniform(0, 2000, n))
        y = np.sin(x) + 0.1 * rng.normal(size=n)
        gp = george.GP(1.0 * kernels.Matern32Kernel(4.0), solver=george.HODLRSolver, min_size=256, tol=1e-10,
                       exhaust="lowrank")
        gp.compute(x, 0.1)
        t = rng.uniform(-5, 2005, 4096)
        recs.append(run("hodlr_m32_1d_n262144", gp, y, t, max(1, a.reps // 2), name_card))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "predict_grad_bench.json"), "w") as fh:
            json.dump(recs, fh, indent=1)


if __name__ == "__main__":
    main()
