# -*- coding: utf-8 -*-
"""HODLRSolver.grad_terms (bgp_hodlr_grad_terms) on its two regimes: K^-1 resident (n <= 65536) and streamed in
column slabs through the row-restricted solve.

    python tools/hodlr_grad_bench.py [--reps 3] [--max-n 262144]

One JSON line per (workload, n, path):
  grad_ms        grad_terms wall time with a device synchronise around it, median of --reps calls
  solve_ms       of one extra call with profiling on, the time in the solves (alpha and K^-1), CUDA events
  contract_ms    of that call, the contraction (with the diagonal and the reductions); with profiling on every slab
                 waits for its events, so solve_ms + contract_ms can exceed grad_ms slightly
  slabs, slab_cols  the streamed path's K^-1 slabs (0 on the resident path)
  max_rel_diff   streamed rows at n <= 65536: max_p |g_stream - g_resident| / |g_resident| on the same handle
  card           GPU name and power limit, read in the same run
Workloads: bench.py's cfg3 (Matern-3/2 1-D, leaf 256, tol 1e-10) and cfg2 (ExpSquared 1-D, min_size 100, tol 1e-10),
both with exhaust="lowrank".  At n = 16384 and 65536 the same handle runs the resident path and then the streamed path
with BGP_GRAD_CHUNK set to the default slab width, so both sides of the selection have a workload; at N = 2^17 and 2^18
the default selection streams.
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
from george_b200 import _lib, kernels  # noqa: E402

WORKLOADS = {
    "cfg3": dict(label="Matern32Kernel 1D leaf=256 tol=1e-10", min_size=256, tol=1e-10,
                 kernel=lambda: 1.0 * kernels.Matern32Kernel(1.0)),
    "cfg2": dict(label="ExpSquaredKernel 1D min_size=100 tol=1e-10", min_size=100, tol=1e-10,
                 kernel=lambda: 1.0 * kernels.ExpSquaredKernel(1.0)),
}


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, universal_newlines=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception:
        return "unknown"


def make_data(n):  # bench.py's inputs
    rng = np.random.default_rng(1234)
    x = np.sort(rng.uniform(0, 10 * n / 1000, n))
    yerr = 0.1 * np.ones(n)
    y = np.sin(x) + 0.1 * rng.normal(size=n)
    return x, yerr, y


def default_cols(n):
    return max(64, (1 << 27) // n // 64 * 64)


def timed(s, y, which, reps):
    lib = _lib.load()
    times = []
    out = None
    for _ in range(reps):
        _lib.check(lib.bgp_dev_synchronize())
        t0 = time.perf_counter()
        out = s.grad_terms(y, which)
        _lib.check(lib.bgp_dev_synchronize())
        times.append(1e3 * (time.perf_counter() - t0))
    s.solver.set_profiling(True)
    s.grad_terms(y, which)
    s.solver.set_profiling(False)
    t = s.solver.grad_timing()
    return out, float(np.median(times)), t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--max-n", type=int, default=1 << 18)
    ap.add_argument("--workload", choices=sorted(WORKLOADS), action="append")
    args = ap.parse_args()
    os.environ.pop("BGP_GRAD_CHUNK", None)
    dev = card()
    for name in args.workload or ["cfg3", "cfg2"]:
        wl = WORKLOADS[name]
        for n in (16384, 65536, 1 << 17, 1 << 18):
            if n > args.max_n:
                continue
            x, yerr, y = make_data(n)
            s = george.HODLRSolver(wl["kernel"](), min_size=wl["min_size"], tol=wl["tol"], seed=42, exhaust="lowrank")
            s.compute(x[:, None], yerr)
            which = np.ones(2, dtype=np.uint32)
            s.grad_terms(y, which)  # warm-up (workspace)
            paths = [("default", None)]
            if n <= 65536:
                paths.append(("streamed", str(default_cols(n))))
            g_res = None
            for path, chunk in paths:
                if chunk:
                    os.environ["BGP_GRAD_CHUNK"] = chunk
                    s.grad_terms(y, which)
                try:
                    (alpha, g, diag), ms, t = timed(s, y, which, args.reps)
                finally:
                    os.environ.pop("BGP_GRAD_CHUNK", None)
                row = {"workload": name, "label": wl["label"], "n": n,
                       "path": "resident" if t["slabs"] == 0 else "streamed", "grad_ms": round(ms, 3),
                       "solve_ms": round(t["solve_ms"], 3), "contract_ms": round(t["contract_ms"], 3),
                       "slabs": t["slabs"], "slab_cols": t["slab_cols"], "card": dev}
                if t["slabs"] == 0:
                    g_res = g
                elif g_res is not None:
                    row["max_rel_diff"] = float(np.max(np.abs(g - g_res) / np.abs(g_res)))
                print(json.dumps(row), flush=True)
            del s


if __name__ == "__main__":
    main()
