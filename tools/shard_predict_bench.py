# -*- coding: utf-8 -*-
"""The sharded HODLR prediction (bgp_hodlr_predict_local_dev) on P = 1, 2, 4, 8 host-exchange shards in ONE process on
one GPU, against the unsharded bgp_hodlr_predict at the same N.

    python tools/shard_predict_bench.py [--reps 3] [--n 262144] [--shards 1 2 4 8]

Each shard is a handle computed with shard_rank = s, shard_count = P and finished by the host's exchange
(shard_grad_bench.shards).  For each kind, B = K(x, x*) is built on the device, every shard solves it with the split
solve (solve_local_dev, its rows gathered into one device block, solve_top_dev on a copy of that block), and that
shard's local prediction is timed on its own W, with the prior on shard 0.  The shards run one after another on the
same GPU, so the largest per-shard time stands in for the P-GPU prediction time MINUS the chunks' solves and the final
all-reduce (ns or ns^2 doubles), which are not measured here.  One JSON line per (kind, run):
  kind, ns        "var" at ns = 4096 or "cov" at ns = 1024
  run             "single" (unsharded bgp_hodlr_predict, solve included) or "shards"
  predict_ms      single: bgp_hodlr_predict wall time, median of --reps synchronised calls after one warm-up call;
                  predict_spread_ms = [min, max]
  shard_ms        shards: each shard's predict_local wall time (the solve excluded), median of --reps synchronised
                  calls after a warm-up call; shard_spread_ms = [min, max] per shard
  max_shard_ms    the largest of shard_ms
  rel_diff        max |sum of the shard parts - single| / max |K**|  (the prior's scale, as tests/test_gpu_predict.py)
  card            GPU name and power limit, read in the same run
Workload: bench.py's cfg3 (Matern-3/2 1-D, leaf 256, tol 1e-10) with exhaust="lowrank", bench.py's inputs, and test
points drawn uniformly over the range of x.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import shard_grad_bench as sgb  # noqa: E402
from george_b200 import _lib, kernels  # noqa: E402
from george_b200._spec import flatten  # noqa: E402
from george_b200.solvers._hodlr import HODLRSolver as Native  # noqa: E402
from george_b200.solvers.basic import BasicSolver  # noqa: E402

KINDS = [("var", 4096), ("cov", 1024)]


def sync():
    torch.cuda.synchronize()
    sgb.sync()


def timed(fn, reps):
    """(last result, median ms, [min ms, max ms]) of reps synchronised calls after one warm-up call."""
    out = fn()
    times = []
    for _ in range(reps):
        sync()
        t0 = time.perf_counter()
        out = fn()
        sync()
        times.append(1e3 * (time.perf_counter() - t0))
    return out, float(np.median(times)), [round(min(times), 2), round(max(times), 2)]


def build_B(kernel, x_dev, xs):
    """K(x, x*) on the device: (ns, n) row-major = n x ns column-major."""
    n, ns = x_dev.shape[0], xs.shape[0]
    xs_dev = torch.from_numpy(np.ascontiguousarray(xs)).cuda()
    B = torch.empty((ns, n), dtype=torch.float64, device="cuda")
    spec = flatten(kernel)
    sync()
    _lib.check(_lib.load().bgp_kmat_general_dev(C.byref(spec), C.c_void_p(xs_dev.data_ptr()), ns,
                                                C.c_void_p(x_dev.data_ptr()), n, C.c_void_p(B.data_ptr()), n))
    sync()
    return B


def run_single(kernel, x, yerr, xs, kind, reps, dev):
    s = Native()
    s.compute(kernel, x, yerr, sgb.MIN_SIZE, sgb.TOL, 42, rng_mode="pernode", exhaust="lowrank")
    out, ms, spread = timed(lambda: BasicSolver._predictive_call(s._lib.bgp_hodlr_predict, s._ptr, kernel, xs, kind),
                            reps)
    print(json.dumps({"kind": kind, "ns": xs.shape[0], "run": "single", "n": x.shape[0], "predict_ms": round(ms, 2),
                      "predict_spread_ms": spread, "card": dev}), flush=True)
    del s
    Native.release_parked()
    return out


def run_shards(kernel, x, yerr, P, reps, dev, work):
    lib = _lib.load()
    n = x.shape[0]
    hs, ranges = sgb.shards(kernel, x, yerr, P)
    x_dev = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    for kind, xs, ref, kss in work:
        ns = xs.shape[0]
        B = build_B(kernel, x_dev, xs)
        W, T = torch.empty_like(B), torch.empty_like(B)
        for s, (row0, rows) in zip(hs, ranges):  # the split solve's local part, this shard's rows gathered into W
            T.copy_(B)
            sync()
            _lib.check(lib.bgp_hodlr_solve_local_dev(s._ptr, C.c_void_p(T.data_ptr()), ns, n))
            sync()
            W[:, row0:row0 + rows] = T[:, row0:row0 + rows]
        del B
        row = {"kind": kind, "ns": ns, "run": "shards", "n": n, "P": P, "shard_ms": [], "shard_spread_ms": [],
               "card": dev}
        total = None
        for k, s in enumerate(hs):
            T.copy_(W)
            sync()
            _lib.check(lib.bgp_hodlr_solve_top_dev(s._ptr, C.c_void_p(T.data_ptr()), ns, n))
            sync()
            part, ms, spread = timed(lambda: s.predict_local(kernel, xs, kind, C.c_void_p(T.data_ptr()), n, k == 0),
                                     reps)
            total = part if total is None else total + part
            row["shard_ms"].append(round(ms, 2))
            row["shard_spread_ms"].append(spread)
        del W, T
        row["max_shard_ms"] = max(row["shard_ms"])
        row["rel_diff"] = float(np.max(np.abs(total - ref)) / np.max(np.abs(kss)))
        print(json.dumps(row), flush=True)
    del hs
    Native.release_parked()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--n", type=int, default=1 << 18)
    ap.add_argument("--shards", type=int, nargs="*", default=[1, 2, 4, 8])
    args = ap.parse_args()
    os.environ.pop("BGP_PREDICT_CHUNK", None)
    dev = sgb.card()
    kernel = 1.0 * kernels.Matern32Kernel(1.0)
    x, yerr, _ = sgb.make_data(args.n)
    rng = np.random.default_rng(4321)
    work = []
    for kind, ns in KINDS:
        xs = rng.uniform(x.min() - 0.5, x.max() + 0.5, (ns, 1))
        kss = kernel.get_value(xs, diag=True) if kind == "var" else kernel.get_value(xs)
        work.append((kind, xs, run_single(kernel, x, yerr, xs, kind, args.reps, dev), kss))
    for P in args.shards:
        run_shards(kernel, x, yerr, P, args.reps, dev, work)


if __name__ == "__main__":
    main()
