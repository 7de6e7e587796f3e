# -*- coding: utf-8 -*-
"""The sharded HODLR prediction (bgp_hodlr_predict_local_dev) and its variance gradient
(bgp_hodlr_predict_grad_local_dev) on P = 1, 2, 4, 8 host-exchange shards in ONE process on one GPU, against the
unsharded bgp_hodlr_predict / bgp_hodlr_predict_grad at the same N.

    python tools/shard_predict_bench.py [--reps 3] [--n 262144] [--shards 1 2 4 8] [--kinds var cov grad]
                                        [--host-ns 512]

Each shard is a handle computed with shard_rank = s, shard_count = P and finished by the host's exchange
(shard_grad_bench.shards).  For each kind, B = K(x, x*) is built on the device, every shard solves it with the split
solve (solve_local_dev, its rows gathered into one device block, solve_top_dev on a copy of that block), and that
shard's local prediction is timed on its own W, with the prior on shard 0.  The shards run one after another on the
same GPU, so the largest per-shard time stands in for the P-GPU prediction time MINUS the chunks' solves and the final
all-reduce(s) (ns or ns^2 doubles; for grad ns and then ns * ndim), which are not measured here.  --kinds selects the
kinds (default var and cov).  One JSON line per (kind, run):
  kind, ns        "var" at ns = 4096, "cov" at ns = 1024 or "grad" (var and dvar) at ns = 4096
  run             "single" (unsharded bgp_hodlr_predict / bgp_hodlr_predict_grad, solve included) or "shards"
  predict_ms      single: the unsharded call's wall time, median of --reps synchronised calls after one warm-up call;
                  predict_spread_ms = [min, max]
  shard_ms        shards: each shard's predict_local / predict_grad_local wall time (the solve excluded), median of
                  --reps synchronised calls after a warm-up call; shard_spread_ms = [min, max] per shard
  max_shard_ms    the largest of shard_ms
  rel_diff        max |sum of the shard parts - single| / max |K**|  (the prior's scale, as tests/test_gpu_predict.py;
                  for grad the larger of var's and dvar's)
  card            GPU name and power limit, read in the same run
With grad, one more line, run "host_route", at ns = --host-ns (the host route holds ns x N doubles several times over):
the route a sharded GP.grad_predict(return_var=True) took before the collective bgp_hodlr_predict_grad, on an unsharded
handle: K(x*, x) to the host, apply_inverse of its transpose (host copies in and out), the variance on the host and
x1_gradient_matvec uploading the solve again.  host_ms is its wall time, device_ms bgp_hodlr_predict_grad's at the same
ns (both medians as above), rel_diff the two routes' difference on the prior's scale.
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
from george_b200.gp import GP  # noqa: E402
from george_b200.solvers._hodlr import HODLRSolver as Native  # noqa: E402
from george_b200.solvers.basic import BasicSolver  # noqa: E402

KINDS = [("var", 4096), ("cov", 1024), ("grad", 4096)]


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


def single_call(s, kernel, xs, kind):
    """The unsharded prediction of one kind: out, or (var, dvar) for grad."""
    if kind == "grad":
        return BasicSolver._predictive_grad_call(s._lib.bgp_hodlr_predict_grad, s._ptr, kernel, xs)
    return BasicSolver._predictive_call(s._lib.bgp_hodlr_predict, s._ptr, kernel, xs, kind)


def rel_diff(got, ref, kss):
    got, ref = (got, ref) if isinstance(ref, tuple) else ((got,), (ref,))
    return float(max(np.max(np.abs(g - r)) for g, r in zip(got, ref)) / np.max(np.abs(kss)))


def run_single(kernel, x, yerr, xs, kind, reps, dev):
    s = Native()
    s.compute(kernel, x, yerr, sgb.MIN_SIZE, sgb.TOL, 42, rng_mode="pernode", exhaust="lowrank")
    out, ms, spread = timed(lambda: single_call(s, kernel, xs, kind), reps)
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
            w_dev = C.c_void_p(T.data_ptr())
            if kind == "grad":
                part, ms, spread = timed(lambda: s.predict_grad_local(kernel, xs, w_dev, n, k == 0), reps)
                total = part if total is None else (total[0] + part[0], total[1] + part[1])
            else:
                part, ms, spread = timed(lambda: s.predict_local(kernel, xs, kind, w_dev, n, k == 0), reps)
                total = part if total is None else total + part
            row["shard_ms"].append(round(ms, 2))
            row["shard_spread_ms"].append(spread)
        del W, T
        row["max_shard_ms"] = max(row["shard_ms"])
        row["rel_diff"] = rel_diff(total, ref, kss)
        print(json.dumps(row), flush=True)
    del hs
    Native.release_parked()


def run_host_route(kernel, x, yerr, xs, reps, dev):
    s = Native()
    s.compute(kernel, x, yerr, sgb.MIN_SIZE, sgb.TOL, 42, rng_mode="pernode", exhaust="lowrank")

    def host():
        Kxs = kernel.get_value(xs, x)
        KinvKxs = s.apply_inverse(Kxs.T)
        return (GP._host_var(Kxs, KinvKxs, xs, kernel),
                kernel.kernel.x1_gradient_matvec(xs, x, KinvKxs, scale=-2.0, add_prior=True))

    got, host_ms, host_spread = timed(host, reps)
    ref, dev_ms, dev_spread = timed(lambda: single_call(s, kernel, xs, "grad"), reps)
    print(json.dumps({"kind": "grad", "ns": xs.shape[0], "run": "host_route", "n": x.shape[0],
                      "host_ms": round(host_ms, 2), "host_spread_ms": host_spread, "device_ms": round(dev_ms, 2),
                      "device_spread_ms": dev_spread, "rel_diff": rel_diff(got, ref, kernel.get_value(xs, diag=True)),
                      "card": dev}), flush=True)
    del s
    Native.release_parked()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--n", type=int, default=1 << 18)
    ap.add_argument("--shards", type=int, nargs="*", default=[1, 2, 4, 8])
    ap.add_argument("--kinds", nargs="*", choices=[k for k, _ in KINDS], default=["var", "cov"])
    ap.add_argument("--host-ns", type=int, default=512)
    args = ap.parse_args()
    os.environ.pop("BGP_PREDICT_CHUNK", None)
    dev = sgb.card()
    kernel = 1.0 * kernels.Matern32Kernel(1.0)
    x, yerr, _ = sgb.make_data(args.n)
    rng = np.random.default_rng(4321)
    work = []
    for kind, ns in KINDS:  # every kind's points are drawn, so a kind's points do not depend on --kinds
        xs = rng.uniform(x.min() - 0.5, x.max() + 0.5, (ns, 1))
        if kind not in args.kinds:
            continue
        kss = kernel.get_value(xs) if kind == "cov" else kernel.get_value(xs, diag=True)
        work.append((kind, xs, run_single(kernel, x, yerr, xs, kind, args.reps, dev), kss))
    if "grad" in args.kinds:
        run_host_route(kernel, x, yerr, rng.uniform(x.min() - 0.5, x.max() + 0.5, (args.host_ns, 1)), args.reps, dev)
    for P in args.shards:
        run_shards(kernel, x, yerr, P, args.reps, dev, work)


if __name__ == "__main__":
    main()
