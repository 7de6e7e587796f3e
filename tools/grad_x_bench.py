# -*- coding: utf-8 -*-
"""GP.grad_log_likelihood_x(..., return_gradient=True) against GP.grad_log_likelihood on the same GP.

    python tools/grad_x_bench.py [--reps 5] [--dense 4096 16384] [--hodlr 65536 131072 262144] [--shards 4]

One JSON line per workload and size:
  grad_s, grad_x_s      median wall time of --reps synchronised calls (after one warm-up call each), seconds;
                        *_spread_s = [min, max]
  ratio                 grad_x_s / grad_s
  grad_rel, grad_self_rel   max relative difference of the returned grad from a grad_log_likelihood call, and of two
                        grad_log_likelihood calls from each other (0 where the solver's sums are reproducible: dense,
                        and HODLR up to N = 1024, whose solve sums with atomics above)
  card                  GPU name and power limit, read in the same run
Workloads: "dense" (BasicSolver, Matern-3/2 1-D, bench.py's inputs) and "hodlr_cfg3" (bench.py's cfg3: Matern-3/2 1-D,
leaf 256, tol 1e-10, exhaust="lowrank"; resident at N = 65536, streamed above).  --shards P adds, at the largest HODLR
size, P host-exchange shards on the one GPU, timed as tools/shard_grad_bench.py does: each shard's local call
(bgp_hodlr_grad_terms_local_dev, then bgp_hodlr_grad_x_terms_local_dev) on its own, the slowest shard reported
(max_shard_grad_s, max_shard_grad_x_s); the alpha solve and the collectives are not in it.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import george_b200 as george  # noqa: E402
from george_b200 import kernels  # noqa: E402
from george_b200.solvers import HODLRSolver  # noqa: E402
from george_b200.solvers._hodlr import HODLRSolver as Native  # noqa: E402
import shard_grad_bench as sgb  # noqa: E402


def timed(fn, reps):
    fn()
    times = []
    for _ in range(reps):
        sgb.sync()
        t0 = time.perf_counter()
        fn()
        sgb.sync()
        times.append(time.perf_counter() - t0)
    return float(np.median(times)), [round(min(times), 4), round(max(times), 4)]


def run_gp(workload, n, reps, card):
    x, yerr, y = sgb.make_data(n)
    k = 1.0 * kernels.Matern32Kernel(1.0)
    if workload == "dense":
        gp = george.GP(k)
    else:
        gp = george.GP(k, solver=HODLRSolver, min_size=sgb.MIN_SIZE, tol=sgb.TOL, exhaust="lowrank")
    gp.compute(x[:, 0], yerr)
    g_s, g_sp = timed(lambda: gp.grad_log_likelihood(y), reps)
    x_s, x_sp = timed(lambda: gp.grad_log_likelihood_x(y, return_gradient=True), reps)
    ref, again = gp.grad_log_likelihood(y), gp.grad_log_likelihood(y)
    got = gp.grad_log_likelihood_x(y, return_gradient=True)[0]
    print(json.dumps({"workload": workload, "n": n, "grad_s": round(g_s, 4), "grad_spread_s": g_sp,
                      "grad_x_s": round(x_s, 4), "grad_x_spread_s": x_sp, "ratio": round(x_s / g_s, 3),
                      "grad_rel": float(np.max(np.abs(got - ref) / np.abs(ref))),
                      "grad_self_rel": float(np.max(np.abs(again - ref) / np.abs(ref))), "card": card}), flush=True)
    del gp
    Native.release_parked()


def run_shards(n, P, reps, card):
    x, yerr, y = sgb.make_data(n)
    kernel = 1.0 * kernels.Matern32Kernel(1.0)
    which = np.ones(2, dtype=np.uint32)
    hs, ranges = sgb.shards(kernel, x, yerr, P)
    alphas = sgb.sharded_alpha(hs, ranges, y)
    diag, dx = sgb.Dev(n), sgb.Dev(n)
    g_ms, x_ms = [], []
    for s, a in zip(hs, alphas):
        g_ms.append(timed(lambda: s.grad_terms_local(a.p, which, diag.p), reps)[0])
        x_ms.append(timed(lambda: s.grad_x_terms_local(a.p, which, dx.p, diag.p), reps)[0])
    print(json.dumps({"workload": "hodlr_cfg3_shards", "n": n, "P": P, "shard_grad_s": [round(t, 4) for t in g_ms],
                      "shard_grad_x_s": [round(t, 4) for t in x_ms], "max_shard_grad_s": round(max(g_ms), 4),
                      "max_shard_grad_x_s": round(max(x_ms), 4), "ratio": round(max(x_ms) / max(g_ms), 3),
                      "card": card}), flush=True)
    del hs, alphas
    Native.release_parked()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--dense", type=int, nargs="*", default=[4096, 16384])
    ap.add_argument("--hodlr", type=int, nargs="*", default=[1 << 16, 1 << 17, 1 << 18])
    ap.add_argument("--shards", type=int, nargs="*", default=[4])
    args = ap.parse_args()
    os.environ.pop("BGP_GRAD_CHUNK", None)
    card = sgb.card()
    for n in args.dense:
        run_gp("dense", n, args.reps, card)
    for n in args.hodlr:
        run_gp("hodlr_cfg3", n, args.reps, card)
    if args.hodlr:
        for P in args.shards:
            run_shards(max(args.hodlr), P, args.reps, card)


if __name__ == "__main__":
    main()
