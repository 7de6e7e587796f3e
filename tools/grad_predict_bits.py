# -*- coding: utf-8 -*-
"""Seeded outputs of GP.grad_predict (with and without return_var) and GP.predict(return_var=True) on dense models,
saved as .npy, to show that two builds of the predictive-gradient code produce the same bits.

    python tools/grad_predict_bits.py save OUTDIR        # on the device: one .npy per (model, n, ns, return_var)
    python tools/grad_predict_bits.py compare DIR1 DIR2  # on any machine: every file of DIR1 equal, bit for bit, in DIR2

Models: Matern-3/2 1-D (the specialised input-gradient evaluator) and ExpSquared 3-D with a general metric (the
interpreter) at n = 65 and 1000; ns = 1, 9 and 300 (either side of the few-column step kernels of the backward sweep).
Each file holds mu, dmu (and var, dvar) of grad_predict followed by predict's mu and var, flattened.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

MODELS = ("m32_1d", "expsq_3d_general")
TEST_SIZES = (1, 9, 300)
CASES = [(m, n, ns, rv) for m in MODELS for n in (65, 1000) for ns in TEST_SIZES for rv in (False, True)]


def _model(name, n):
    import george_b200 as george
    from george_b200 import kernels
    rng = np.random.default_rng(n)
    if name == "m32_1d":
        x = np.sort(rng.uniform(0, 10, n))
        y = np.sin(x) + 0.1 * rng.standard_normal(n)
        gp = george.GP(1.7 * kernels.Matern32Kernel(0.8), mean=0.2)
        t = lambda ns: np.linspace(-1, 11, ns)  # noqa: E731
    else:
        x = rng.uniform(-2, 2, (n, 3))
        y = np.sin(x[:, 0]) * np.cos(x[:, 1]) + 0.1 * rng.standard_normal(n)
        metric = [[1.0, 0.1, 0.2], [0.1, 2.0, 0.3], [0.2, 0.3, 1.5]]
        gp = george.GP(0.9 * kernels.ExpSquaredKernel(metric, ndim=3), mean=-0.1)
        t = lambda ns: np.random.default_rng(ns).uniform(-2.5, 2.5, (ns, 3))  # noqa: E731
    gp.compute(x, 0.1)
    return gp, y, t


def save(outdir):
    os.makedirs(outdir, exist_ok=True)
    for name, n, ns, rv in CASES:
        gp, y, t = _model(name, n)
        ts = t(ns)
        out = list(gp.grad_predict(y, ts, return_var=rv)) + list(gp.predict(y, ts, return_var=True))
        np.save(os.path.join(outdir, "%s_%d_%d_%d.npy" % (name, n, ns, rv)),
                np.concatenate([np.ravel(a) for a in out]))
    print("saved %d files to %s" % (len(CASES), outdir))


def compare(d1, d2):
    names = sorted(f for f in os.listdir(d1) if f.endswith(".npy"))
    assert len(names) == len(CASES), names
    for f in names:
        a, b = np.load(os.path.join(d1, f)), np.load(os.path.join(d2, f))
        same = a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))
        print("%-34s %s" % (f, "equal" if same else "DIFFERENT"))
        assert same, f
    print("all %d files equal" % len(names))


if __name__ == "__main__":
    if sys.argv[1] == "save":
        save(sys.argv[2])
    else:
        compare(sys.argv[2], sys.argv[3])
