# -*- coding: utf-8 -*-
"""The sharded HODLR symmetric factor K~ = W W^T (bgp_hodlr_sym_factor_local / _finish_top, bgp_hodlr_sym_apply_*_dev)
on P = 1, 2, 4, 8 host-exchange shards in ONE process on one GPU, against the unsharded build at the same N.

    python tools/shard_sqrt_bench.py [--reps 3] [--n 262144] [--shards 1 2 4 8] [--nrhs 64]

Each shard is a handle computed with shard_rank = s, shard_count = P and finished by the host's exchange
(shard_grad_bench.shards).  The factor is then built step by step: every shard's local part, the host's exchange of the
top columns' rows (sym_export_top, sym_import_top), every shard's finish; and W Z is applied to --nrhs standard normal
columns (top, local, the host assembling the rows).  The shards run one after another on the same GPU, so the largest
per-shard time stands in for the P-GPU time MINUS the all-gathers (of the top columns' rows in the build, of each
64-column group's rows in the apply), which are not measured here.  One JSON line per run:
  run             "single" (unsharded: bgp_hodlr_sym_factor and bgp_hodlr_sym_apply) or "shards"
  build_ms        single: the build's wall time (factor_local + finish_top on the unsharded handle: the whole factor),
                  median of --reps synchronised builds after one warm-up; build_spread_ms = [min, max]
  apply_ms        single: W Z on a device block (apply_local_dev: all of W), median as above
  local_ms, finish_ms, apply_ms   shards: per shard, the local build, the finish (the top levels over all N rows) and
                  the apply (top + local on a device block), medians as above
  max_local_ms, max_finish_ms, max_apply_ms   the largest over the shards
  logdet_rel      |sum of the partial log|K~| - single| / |single|
  apply_rel       max |W Z (shards) - W Z (single)| / max |W Z (single)|
  card            GPU name and power limit, read in the same run
Workload: bench.py's cfg3 (Matern-3/2 1-D, leaf 256, tol 1e-10) with exhaust="lowrank" and bench.py's inputs.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import shard_grad_bench as sgb  # noqa: E402
from george_b200 import _lib, kernels  # noqa: E402
from george_b200.solvers._hodlr import HODLRSolver as Native  # noqa: E402


def build(hs, ranges, cols):
    """The step-by-step build on every shard: (partial log-dets, per-shard local ms, per-shard finish ms); the
    exchange between them is not timed."""
    rows_pad = max(r for _, r in ranges)
    local, finish = [], []
    for s in hs:
        sgb.sync()
        t0 = time.perf_counter()
        s.symmetric_factor_local()
        sgb.sync()
        local.append(1e3 * (time.perf_counter() - t0))
    buf = sgb.Dev(len(hs) * max(cols, 1) * rows_pad)
    for r, s in enumerate(hs):
        s.symmetric_export_top(buf.at(r * cols * rows_pad), rows_pad)
    sgb.sync()
    for s in hs:
        s.symmetric_import_top(buf.p, rows_pad)
    partial = []
    for s in hs:
        sgb.sync()
        t0 = time.perf_counter()
        partial.append(s.symmetric_finish_top())
        sgb.sync()
        finish.append(1e3 * (time.perf_counter() - t0))
    return partial, local, finish


def top_cols(s, P):
    """The top panel's columns of a shard (0 on an unsharded handle)."""
    if P == 1:
        return 0
    ptr, row0, rows, cols, ld = C.c_void_p(), C.c_int64(), C.c_int64(), C.c_int64(), C.c_int64()
    _lib.check(s._lib.bgp_hodlr_top_panel(s._ptr, C.byref(ptr), C.byref(row0), C.byref(rows), C.byref(cols),
                                          C.byref(ld)))
    return cols.value


def median(v):
    return round(float(np.median(v)), 2), [round(min(v), 2), round(max(v), 2)]


def apply_shards(hs, ranges, Z, n):
    """W Z on the shards (top, local, the host's assembly of the rows); (result, per-shard ms of top + local)."""
    k = Z.shape[1]
    out = np.empty((k, n))
    ms = []
    buf = sgb.Dev(k * n)
    for s, (row0, rows) in zip(hs, ranges):
        buf.upload(Z.T)
        sgb.sync()
        t0 = time.perf_counter()
        s.apply_symmetric_factor_top(buf.p, k, n)
        s.apply_symmetric_factor_local(buf.p, k, n)
        sgb.sync()
        ms.append(1e3 * (time.perf_counter() - t0))
        out[:, row0:row0 + rows] = buf.download(k * n).reshape(k, n)[:, row0:row0 + rows]
    return out.T, ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--n", type=int, default=1 << 18)
    ap.add_argument("--shards", type=int, nargs="*", default=[1, 2, 4, 8])
    ap.add_argument("--nrhs", type=int, default=64)
    args = ap.parse_args()
    dev = sgb.card()
    kernel = 1.0 * kernels.Matern32Kernel(1.0)
    x, yerr, _ = sgb.make_data(args.n)
    n = x.shape[0]
    Z = np.random.default_rng(7).standard_normal((n, args.nrhs))
    ref = None
    for P in [1] + [p for p in args.shards if p != 1]:  # the unsharded run first: the reference
        hs, ranges = sgb.shards(kernel, x, yerr, P)
        cols = top_cols(hs[0], P)
        runs = [build(hs, ranges, cols) for _ in range(args.reps + 1)][1:]
        applies = [apply_shards(hs, ranges, Z, n) for _ in range(args.reps + 1)][1:]
        partial = runs[-1][0]
        WZ = applies[-1][0]
        if P == 1:
            ref = (partial[0], WZ)
            b, bs = median([r[1][0] + r[2][0] for r in runs])
            a, as_ = median([ap_[1][0] for ap_ in applies])
            row = {"run": "single", "n": n, "nrhs": args.nrhs, "build_ms": b, "build_spread_ms": bs, "apply_ms": a,
                   "apply_spread_ms": as_, "card": dev}
            print(json.dumps(row), flush=True)
        else:
            row = {"run": "shards", "n": n, "P": P, "nrhs": args.nrhs, "card": dev}
            for key, vals in (("local_ms", [[r[1][i] for r in runs] for i in range(P)]),
                              ("finish_ms", [[r[2][i] for r in runs] for i in range(P)]),
                              ("apply_ms", [[ap_[1][i] for ap_ in applies] for i in range(P)])):
                row[key] = [median(v)[0] for v in vals]
                row["max_" + key] = max(row[key])
            row["logdet_rel"] = abs(sum(partial) - ref[0]) / abs(ref[0])
            row["apply_rel"] = float(np.max(np.abs(WZ - ref[1])) / np.max(np.abs(ref[1])))
            print(json.dumps(row), flush=True)
        del hs
        Native.release_parked()


if __name__ == "__main__":
    main()
