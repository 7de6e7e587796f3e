# -*- coding: utf-8 -*-
"""GP.fisher_information(y) against GP.grad_log_likelihood(y) on the dense solver.

    python tools/fisher_bench.py [--reps 5] [--matern 4096 16384] [--co2 512 4096]

One JSON line per workload and size:
  grad_s, fisher_s      median wall time of --reps calls (each call synchronises; one warm-up call each first),
                        seconds; *_spread_s = [min, max]
  ratio                 fisher_s / grad_s
  rows                  kernel rows and white-noise rows of the Fisher pass
  kernel_row_ms, wn_row_ms   median device time of one row's products (CUDA events around the DMMA products of
                        bgp_dense_fisher_terms: the dK_p build, T = K^-1 dK_p and B = K^-1 T^T for a kernel row; the
                        row scaling and K^-1 diag(v) K^-1 for a white-noise row)
  kernel_row_tflops, wn_row_tflops   achieved FP64 rate of those products, from the shapes: 3 n^3 flops per kernel row
                        (2 n^3 for T, n^3 for B's lower triangle), n^3 per white-noise row
  card                  GPU name and power limit, read in the same run
Workloads: "matern32" (bench.py's inputs: Matern-3/2 1-D, yerr = 0.1, fitted amplitude, scale and white noise) and
"co2" (tools/batch_bench.py's CO2 GP: four kernel products, fitted mean and white noise).
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
from batch_bench import card, co2_gp  # noqa: E402


def matern_gp(n):
    rng = np.random.default_rng(1234)  # bench.py's inputs
    x = np.sort(rng.uniform(0, 10 * n / 1000, n))
    y = np.sin(x) + 0.1 * rng.normal(size=n)
    gp = george.GP(1.0 * kernels.Matern32Kernel(1.0), white_noise=np.log(0.01), fit_white_noise=True)
    gp.compute(x, 0.1)
    return gp, y


def timed(fn, reps):
    fn()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t0)
    return float(np.median(times)), [round(min(times), 4), round(max(times), 4)]


def row_times(gp, reps):
    """Median device ms of each row's products over ``reps`` calls of the solver hook, kernel rows then white-noise
    rows (the GP's white-noise vectors v_k = exp(wn) dwn_k)."""
    mask = gp.kernel.unfrozen_mask.astype(np.uint32)
    v = np.zeros((0, len(gp._x)))
    if len(gp.white_noise):
        wn, dwn = gp._white_noise_terms()
        v = np.exp(wn)[None, :] * dwn
    nk = int(mask.sum())
    ms = np.zeros((reps, nk + v.shape[0]))
    for r in range(reps):
        gp.solver.fisher_terms(None, mask, v, prod_ms=ms[r])
    med = np.median(ms, axis=0)
    return med[:nk], med[nk:]


def run(workload, n, reps, gpu_card):
    gp, y = matern_gp(n) if workload == "matern32" else co2_gp(n)[:2]
    n = len(gp._x)
    g_s, g_sp = timed(lambda: gp.grad_log_likelihood(y), reps)
    f_s, f_sp = timed(lambda: gp.fisher_information(y), reps)
    grad, F = gp.fisher_information(y)
    k_ms, w_ms = row_times(gp, reps)
    out = dict(workload=workload, n=n, params=len(gp), rows=[len(k_ms), len(w_ms)], grad_s=round(g_s, 4),
               grad_spread_s=g_sp, fisher_s=round(f_s, 4), fisher_spread_s=f_sp, ratio=round(f_s / g_s, 2),
               grad_bit_equal=bool(np.array_equal(grad, gp.grad_log_likelihood(y))),
               symmetric=bool(np.array_equal(F, F.T)))
    if len(k_ms):
        km = float(np.median(k_ms))
        out.update(kernel_row_ms=round(km, 2), kernel_row_tflops=round(3.0 * n ** 3 / (km * 1e-3) / 1e12, 2))
    if len(w_ms):
        wm = float(np.median(w_ms))
        out.update(wn_row_ms=round(wm, 2), wn_row_tflops=round(1.0 * n ** 3 / (wm * 1e-3) / 1e12, 2))
    out["card"] = gpu_card
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--matern", type=int, nargs="*", default=[4096, 16384])
    ap.add_argument("--co2", type=int, nargs="*", default=[512, 4096])
    args = ap.parse_args()
    gpu_card = card()
    for n in args.matern:
        run("matern32", n, args.reps, gpu_card)
    for n in args.co2:
        run("co2", n, args.reps, gpu_card)


if __name__ == "__main__":
    main()
