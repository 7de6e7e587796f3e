# -*- coding: utf-8 -*-
"""Seeded outputs of the unsharded HODLR symmetric factor, saved as .npy, to show that two builds of the factor's code
produce the same bits.

    python tools/sym_bits.py save OUTDIR        # on the device: one .npy per case
    python tools/sym_bits.py compare DIR1 DIR2  # on any machine: every file of DIR1 equal, bit for bit, in DIR2

Each file holds W(I), W^T(I) (HODLRSolver.apply_symmetric_factor of the identity) and symmetric_log_determinant,
flattened.  Cases: Matern-3/2 and the quasi-periodic kernel at N = 1000 and 1537 (leaf 64, lowrank), and ExpSquared
with a general 2-D metric at N = 1200.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CASES = [("m32", 1000), ("m32", 1537), ("quasiperiodic", 1000), ("quasiperiodic", 1537), ("general2d", 1200)]


def _case(name, n):
    from george_b200 import kernels as K
    from george_b200.solvers._hodlr import HODLRSolver
    rng = np.random.default_rng(3)
    kernel = {"m32": 1.0 * K.Matern32Kernel(1.0),
              "quasiperiodic": 1.0 * K.ExpSquaredKernel(1.0) + 0.5 * K.ExpSine2Kernel(gamma=1.0, log_period=np.log(3.0)),
              "general2d": 1.0 * K.ExpSquaredKernel([[4.0, 0.6], [0.6, 2.0]], ndim=2)}[name]
    if name == "general2d":
        x = rng.uniform(0, 4, (n, 2))
        x = x[np.argsort(x[:, 0])]
    else:
        x = np.sort(rng.uniform(0, 10 * n / 1000, n))[:, None]
    yerr = 0.1 + 0.05 * np.random.default_rng(1).uniform(size=n)
    s = HODLRSolver()
    s.compute(kernel, x, yerr, min_size=64, tol=1e-12, exhaust="lowrank")
    return s


def save(outdir):
    os.makedirs(outdir, exist_ok=True)
    for name, n in CASES:
        s = _case(name, n)
        W = s.apply_symmetric_factor(np.eye(n))
        Wt = s.apply_symmetric_factor(np.eye(n), transpose=True)
        np.save(os.path.join(outdir, "%s_%d.npy" % (name, n)),
                np.concatenate([W.ravel(), Wt.ravel(), [s.symmetric_log_determinant]]))
    print("saved %d files to %s" % (len(CASES), outdir))


def compare(d1, d2):
    names = sorted(f for f in os.listdir(d1) if f.endswith(".npy"))
    assert len(names) == len(CASES), names
    for f in names:
        a, b = np.load(os.path.join(d1, f)), np.load(os.path.join(d2, f))
        same = a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))
        print("%-24s %s" % (f, "equal" if same else "DIFFERENT"))
        assert same, f
    print("all %d files equal" % len(names))


if __name__ == "__main__":
    if sys.argv[1] == "save":
        save(sys.argv[2])
    else:
        compare(sys.argv[2], sys.argv[3])
