# -*- coding: utf-8 -*-
"""The sharded HODLR gradient (bgp_hodlr_grad_terms_local_dev) on P = 1, 2, 4, 8 host-exchange shards in ONE process
on one GPU, against the unsharded streamed bgp_hodlr_grad_terms at the same N.

    python tools/shard_grad_bench.py [--reps 3] [--n 262144] [--shards 1 2 4 8] [--big]

Each shard is a handle computed with shard_rank = s, shard_count = P; the host runs the exchange (export_top, import_top,
finish_top) and the split solve for alpha (solve_local_dev, host assembly, solve_top_dev), then times every shard's local
gradient on its own.  The shards run one after another on the same GPU, so the largest per-shard time stands in for the
P-GPU gradient time MINUS the alpha solve and the two collectives (an all-reduce of P doubles, an all-gather of the diag
slices), which are not measured here.  One JSON line per run:
  kind            "single" (unsharded grad_terms, default selection: streamed above N = 65536) or "shards"
  grad_ms         single: grad_terms wall time, median of --reps synchronised calls after one warm-up call (which
                  also allocates the slab workspace); grad_spread_ms = [min, max] of those calls
  shard_ms        shards: each shard's local gradient wall time, median of --reps synchronised calls after a warm-up
                  call; shard_spread_ms = [min, max] per shard
  max_shard_ms    the largest of shard_ms; ratio = single grad_ms / max_shard_ms
  solve_ms, contract_ms   CUDA-event sums of one more call with profiling on (per shard for "shards")
  slabs, slab_cols        K^-1 slabs of each shard (of the single handle) and their width
  rel_diff        max_p |sum of the shard partials - g_single| / |g_single|
  alpha_rel, diag_rel, log_det_rel   the largest over the shards of each shard's alpha (split solve), the assembled
                  diag and the sum of the partial log-determinants against the single handle's (relative 2-norm /
                  relative difference)
  card            GPU name and power limit, read in the same run
Workload: bench.py's cfg3 (Matern-3/2 1-D, leaf 256, tol 1e-10) with exhaust="lowrank" and bench.py's inputs.  --big adds
P = 8 at N = 2^20 (without the unsharded reference, which would take as long as all eight shards together).
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from george_b200 import _lib, kernels  # noqa: E402
from george_b200.solvers._hodlr import HODLRSolver as Native  # noqa: E402

MIN_SIZE, TOL = 256, 1e-10


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
    return x[:, None], yerr, y


class Dev(object):
    """float64 device buffer from the library's allocator."""

    def __init__(self, count):
        self.lib = _lib.load()
        self.p = C.c_void_p()
        _lib.check(self.lib.bgp_dev_alloc(C.byref(self.p), 8 * max(int(count), 1)))

    def at(self, offset):
        return C.c_void_p(self.p.value + 8 * int(offset))

    def upload(self, a):
        a = np.ascontiguousarray(a, dtype=np.float64)
        _lib.check(self.lib.bgp_dev_upload(self.p, _lib.ptr(a), a.nbytes))

    def download(self, count):
        out = np.empty(count, dtype=np.float64)
        _lib.check(self.lib.bgp_dev_download(_lib.ptr(out), self.p, out.nbytes))
        return out

    def __del__(self):
        if self.p:
            self.lib.bgp_dev_free(self.p)
            self.p = C.c_void_p()


def sync():
    _lib.check(_lib.load().bgp_dev_synchronize())


def shards(kernel, x, yerr, P):
    """P host-exchange shards on newly created handles, computed and finished: (handles, [(row0, rows)])."""
    lib = _lib.load()
    Native.release_parked()
    if P == 1:  # an unsharded handle: its own rows are all N
        s = Native()
        s.compute(kernel, x, yerr, MIN_SIZE, TOL, 42, rng_mode="pernode", exhaust="lowrank")
        return [s], [(0, x.shape[0])]
    hs = []
    for r in range(P):
        s = Native()
        s.compute(kernel, x, yerr, MIN_SIZE, TOL, 42, rng_mode="pernode", shard_rank=r, shard_count=P,
                  exhaust="lowrank")
        hs.append(s)
    ranges = []
    for r in range(P):
        row0, rows = C.c_int64(), C.c_int64()
        _lib.check(lib.bgp_hodlr_shard_rows(hs[0]._ptr, r, C.byref(row0), C.byref(rows)))
        ranges.append((row0.value, rows.value))
    ptr, row0, rows, cols, ld = C.c_void_p(), C.c_int64(), C.c_int64(), C.c_int64(), C.c_int64()
    _lib.check(lib.bgp_hodlr_top_panel(hs[0]._ptr, C.byref(ptr), C.byref(row0), C.byref(rows), C.byref(cols),
                                       C.byref(ld)))
    rows_pad = max(r for _, r in ranges)
    buf = Dev(P * cols.value * rows_pad)
    for r, s in enumerate(hs):
        _lib.check(lib.bgp_hodlr_export_top(s._ptr, buf.at(r * cols.value * rows_pad), rows_pad))
    sync()
    for s in hs:  # bgp.h's call order: every shard imports, then every shard finishes
        _lib.check(lib.bgp_hodlr_import_top(s._ptr, buf.p, rows_pad))
    for s in hs:
        _lib.check(lib.bgp_hodlr_finish_top(s._ptr))
    return hs, ranges


def sharded_alpha(hs, ranges, y):
    """K^-1 y by the split solve; one device copy of the solution per shard."""
    lib = _lib.load()
    n = y.size
    bufs = [Dev(n) for _ in hs]
    if len(hs) == 1:
        bufs[0].upload(hs[0].apply_inverse(y)[:, 0])
        return bufs
    for s, b in zip(hs, bufs):
        b.upload(y)
        _lib.check(lib.bgp_hodlr_solve_local_dev(s._ptr, b.p, 1, n))
    asm = np.empty(n)
    for (row0, rows), b in zip(ranges, bufs):
        asm[row0:row0 + rows] = b.download(n)[row0:row0 + rows]
    for s, b in zip(hs, bufs):
        b.upload(asm)
        _lib.check(lib.bgp_hodlr_solve_top_dev(s._ptr, b.p, 1, n))
    return bufs


def timed(fn, reps):
    """(last result, median ms, [min ms, max ms]) of reps synchronised calls after one warm-up call."""
    times = []
    out = fn()
    for _ in range(reps):
        sync()
        t0 = time.perf_counter()
        out = fn()
        sync()
        times.append(1e3 * (time.perf_counter() - t0))
    return out, float(np.median(times)), [round(min(times), 2), round(max(times), 2)]


def profiled(native, fn):
    native.set_profiling(True)
    fn()
    native.set_profiling(False)
    return native.grad_timing()


def run_single(kernel, x, yerr, y, which, reps, dev):
    s = Native()
    s.compute(kernel, x, yerr, MIN_SIZE, TOL, 42, rng_mode="pernode", exhaust="lowrank")
    n = y.size
    alpha, g, diag = np.empty(n), np.zeros(which.size), np.empty(n)

    def call():
        _lib.check(s._lib.bgp_hodlr_grad_terms(s._ptr, _lib.ptr(which), _lib.ptr(y), _lib.ptr(alpha), _lib.ptr(g),
                                               _lib.ptr(diag)))
        return g.copy()

    g1, ms, spread = timed(call, reps)
    ref = {"g": g1, "alpha": alpha.copy(), "diag": diag.copy(), "log_det": s.log_determinant}
    t = profiled(s, call)
    print(json.dumps({"kind": "single", "n": n, "grad_ms": round(ms, 2), "grad_spread_ms": spread, "solve_ms": round(t["solve_ms"], 2),
                      "contract_ms": round(t["contract_ms"], 2), "slabs": t["slabs"], "slab_cols": t["slab_cols"],
                      "card": dev}), flush=True)
    return ref, ms


def rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def run_shards(kernel, x, yerr, y, which, P, reps, dev, ref=None, single_ms=None):
    hs, ranges = shards(kernel, x, yerr, P)
    alphas = sharded_alpha(hs, ranges, y)
    n = y.size
    diag = Dev(n)
    assembled = np.empty(n)
    row = {"kind": "shards", "n": n, "P": P, "shard_ms": [], "shard_spread_ms": [], "solve_ms": [], "contract_ms": [], "slabs": [],
           "slab_cols": None, "card": dev}
    parts = []
    for s, a in zip(hs, alphas):
        g, ms, spread = timed(lambda: s.grad_terms_local(a.p, which, diag.p), reps)
        t = profiled(s, lambda: s.grad_terms_local(a.p, which, diag.p))
        parts.append(g)
        row0, rows = ranges[len(parts) - 1]
        assembled[row0:row0 + rows] = diag.download(n)[row0:row0 + rows]
        row["shard_ms"].append(round(ms, 2))
        row["shard_spread_ms"].append(spread)
        row["solve_ms"].append(round(t["solve_ms"], 2))
        row["contract_ms"].append(round(t["contract_ms"], 2))
        row["slabs"].append(t["slabs"])
        row["slab_cols"] = t["slab_cols"]
    row["max_shard_ms"] = max(row["shard_ms"])
    if ref is not None:
        g = np.sum(parts, axis=0)
        row["rel_diff"] = float(np.max(np.abs(g - ref["g"]) / np.abs(ref["g"])))
        row["alpha_rel"] = max(rel(a.download(n), ref["alpha"]) for a in alphas)
        row["diag_rel"] = rel(assembled, ref["diag"])
        row["log_det_rel"] = abs(sum(s.log_determinant for s in hs) - ref["log_det"]) / abs(ref["log_det"])
        row["ratio"] = round(single_ms / row["max_shard_ms"], 2)
    print(json.dumps(row), flush=True)
    del hs, alphas
    Native.release_parked()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--n", type=int, default=1 << 18)
    ap.add_argument("--shards", type=int, nargs="*", default=[1, 2, 4, 8])
    ap.add_argument("--big", action="store_true", help="also P = 8 at N = 2^20")
    args = ap.parse_args()
    os.environ.pop("BGP_GRAD_CHUNK", None)
    dev = card()
    kernel = 1.0 * kernels.Matern32Kernel(1.0)
    which = np.ones(2, dtype=np.uint32)
    x, yerr, y = make_data(args.n)
    ref, single_ms = run_single(kernel, x, yerr, y, which, args.reps, dev)
    Native.release_parked()
    for P in args.shards:
        run_shards(kernel, x, yerr, y, which, P, args.reps, dev, ref, single_ms)
    if args.big:
        x, yerr, y = make_data(1 << 20)
        run_shards(kernel, x, yerr, y, which, 8, args.reps, dev)


if __name__ == "__main__":
    main()
