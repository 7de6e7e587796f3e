# -*- coding: utf-8 -*-
"""
Golden vectors of bench.py's ExpSquared (cfg2) and quasi-periodic (cfg5) HODLR workloads at the sizes one GPU runs,
from the CPU oracle in the CUDA path's own mode.

    python tests/golden/make_golden_workloads.py [case ...]       (both cases: under a minute of one core)

Inputs restate bench.py's data law: x = sort(U(0, 10 N / 1000)) from default_rng(1234), yerr = 0.1,
y = sin x + 0.1 N(0, 1).  Solver options as bench.py: min_size = 100, tol = 1e-10, seed = 42, per-node RNG streams
(oracle rng_mode = 0) and exhausted blocks keeping their low-rank factors (exhaust = 1).

    cfg2_fullsize_n65536     1.0 * ExpSquared(1.0),                                  N = 65536
    cfg5_fullsize_n131072    1.0 * ExpSquared(1.0) + 0.5 * ExpSine2(1.0, log 3),     N = 131072 (one GPU's share)

cfg5's eight-GPU size, N = 2^20, has no golden: its unsharded factorisation does not fit one 80 GB device
(tests/test_gpu_zz_workloads.py), and the oracle had not finished it after 25 minutes of one core.

Stored per case: log-determinant, quad = y^T K_h^-1 y, log-likelihood; the oracle's kernel evaluations and the seconds
the run that made the committed file took (CASE_SECONDS: a constant, so that a rerun rebuilds the file bit for bit;
the fresh time is printed); per node (rank, rng draws, dense fallback, is_leaf); the first two pivots (row, col) of
every internal node with their offsets; and a sample of the solve K_h^-1 [y, b] with b = cos(0.37 x): every 64th
row, the 8 rows on each side of every boundary of the eight shards (george_b200.parallel.shard_ranges(N, 8, 100)),
and the first and last 8 rows.

Tests: tests/test_gpu_zz_workloads.py.
"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import oracle  # noqa: E402
from george_b200 import kernels  # noqa: E402
from george_b200._spec import flatten  # noqa: E402
from george_b200.parallel import shard_ranges  # noqa: E402

MIN_SIZE, TOL, SEED = 100, 1e-10, 42
STRIDE, EDGE, SHARDS = 64, 8, 8

CASES = {"cfg2_fullsize_n65536": ("cfg2", 65536), "cfg5_fullsize_n131072": ("cfg5", 131072)}
# seconds of one core (compute, log-det, dot_solve and the two-column solve) of the runs that made the committed files
CASE_SECONDS = {"cfg2_fullsize_n65536": 6.1, "cfg5_fullsize_n131072": 45.7}


def make_kernel(workload):
    if workload == "cfg2":
        return 1.0 * kernels.ExpSquaredKernel(1.0)
    return 1.0 * kernels.ExpSquaredKernel(1.0) + 0.5 * kernels.ExpSine2Kernel(gamma=1.0, log_period=np.log(3.0))


def make_data(n):
    rng = np.random.default_rng(1234)
    x = np.sort(rng.uniform(0, 10 * n / 1000, n))
    yerr = 0.1 * np.ones(n)
    y = np.sin(x) + 0.1 * rng.normal(size=n)
    return x, yerr, y


def second_rhs(x):
    return np.cos(0.37 * x)


def sample_rows(n):
    """Every STRIDE-th row, EDGE rows on each side of every boundary between the SHARDS shards, the first and last
    EDGE rows."""
    idx = [np.arange(0, n, STRIDE), np.arange(EDGE), np.arange(n - EDGE, n)]
    for start, _ in shard_ranges(n, SHARDS, MIN_SIZE)[1:]:
        idx.append(np.arange(start - EDGE, start + EDGE))
    return np.unique(np.concatenate(idx))


def log_likelihood(n, logdet, quad):
    return -0.5 * (n * np.log(2 * np.pi) + logdet) - 0.5 * quad


def make(name):
    workload, n = CASES[name]
    spec = flatten(make_kernel(workload))
    x, yerr, y = make_data(n)
    t0 = time.time()
    h = oracle.HODLR(spec, x, yerr, min_size=MIN_SIZE, tol=TOL, seed=SEED, rng_mode=0, exhaust=1)
    logdet = h.log_determinant
    quad = h.dot_solve(y)
    idx = sample_rows(n)
    sol = h.apply_inverse(np.stack([y, second_rhs(x)], axis=1))[idx]
    secs = time.time() - t0
    nodes = h.nodes()
    info = np.array([[nd["rank"], nd["rng_draws"], nd["dense_fallback"], nd["is_leaf"]] for nd in nodes],
                    dtype=np.int32)
    piv_r, piv_c, piv_off = [], [], [0]
    for i, nd in enumerate(nodes):
        if not nd["is_leaf"]:
            r, c = h.pivots(i, nd["rank"])
            piv_r.extend(r[:2].tolist())
            piv_c.extend(c[:2].tolist())
        piv_off.append(len(piv_r))
    out = dict(n=n, log_determinant=logdet, quad=quad, log_likelihood=log_likelihood(n, logdet, quad),
               oracle_evals=h.num_evals, oracle_seconds=CASE_SECONDS[name],
               node_info=info[:, :3].astype(np.int32), is_leaf=info[:, 3].astype(np.int8),
               piv_rows=np.array(piv_r, dtype=np.int32), piv_cols=np.array(piv_c, dtype=np.int32),
               piv_off=np.array(piv_off, dtype=np.int32), sample_rows=idx.astype(np.int32),
               sample_y=sol[:, 0], sample_b=sol[:, 1])
    print(name, "N", n, "seconds %.1f" % secs, "evals", h.num_evals, "logdet", logdet, "ll", out["log_likelihood"],
          "max rank", int(info[:, 0].max()), flush=True)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), name + ".npz")
    np.savez_compressed(path, **out)
    print("->", path, os.path.getsize(path), "bytes", flush=True)


if __name__ == "__main__":
    for name in sys.argv[1:] or list(CASES):
        make(name)
