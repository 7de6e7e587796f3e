# -*- coding: utf-8 -*-
"""Seeded draws of GP.sample_conditional(rng=g) and utils.device_gaussian_samples, saved as .npy, to show that two
builds of the sampling code produce the same bits.

    python tools/sample_bits.py save OUTDIR        # on the device: one .npy per (route, ns, size)
    python tools/sample_bits.py compare DIR1 DIR2  # on any machine: every file of DIR1 equal, bit for bit, in DIR2

Both product paths are covered (size 1 runs the row kernel, size 16 the DMMA GEMM), at ns = 65 (one ragged tile of
the factorisation) and ns = 1024 (every update level of it).
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CASES = [(ns, size) for ns in (65, 1024) for size in (1, 16)]


def save(outdir):
    import george_b200 as george
    from george_b200 import kernels
    from george_b200.utils import device_gaussian_samples
    os.makedirs(outdir, exist_ok=True)
    rng = np.random.default_rng(0)
    n = 600
    t = np.sort(rng.uniform(0, 30, n))
    y = np.sin(t) + 0.1 * rng.standard_normal(n)
    gp = george.GP(1.0 * kernels.Matern32Kernel(1.0), mean=0.2)
    gp.compute(t, 0.1)
    for ns, size in CASES:
        ts = np.linspace(t[0] - 1, t[-1] + 1, ns)
        d = gp.sample_conditional(y, ts, size, rng=np.random.default_rng(1000 + ns + size))
        np.save(os.path.join(outdir, "cond_%d_%d.npy" % (ns, size)), d)
        q, _ = np.linalg.qr(np.random.default_rng(ns).standard_normal((ns, ns)))
        cov = (q * np.linspace(1.0, 10.0, ns)) @ q.T
        g = np.random.default_rng(2000 + ns + size)
        mean, z = g.standard_normal(ns), g.standard_normal((size, ns))
        np.save(os.path.join(outdir, "mvn_%d_%d.npy" % (ns, size)), device_gaussian_samples(cov, z, mean, 1e-10))
    print("saved %d files to %s" % (2 * len(CASES), outdir))


def compare(d1, d2):
    names = sorted(f for f in os.listdir(d1) if f.endswith(".npy"))
    assert len(names) == 2 * len(CASES), names
    for f in names:
        a, b = np.load(os.path.join(d1, f)), np.load(os.path.join(d2, f))
        same = a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))
        print("%-18s %s" % (f, "equal" if same else "DIFFERENT"))
        assert same, f
    print("all %d files equal" % len(names))


if __name__ == "__main__":
    if sys.argv[1] == "save":
        save(sys.argv[2])
    else:
        compare(sys.argv[2], sys.argv[3])
