# -*- coding: utf-8 -*-
"""
Generates tests/golden/reference_nonfinite.npz by IMPORTING THE REFERENCE (see make_golden.py for the staging): kernel
values and hyper- / x-gradients on non-finite inputs and overflowing parameters, and the dense GP's outcome on broken
problems.  Values are stored as arrays (they hold NaN on purpose), outcomes as strings: "finite", "-inf" or the class
name of the exception ``log_likelihood(y, quiet=False)`` raises.

Run from the repo root:   python tests/golden/make_golden_nonfinite.py
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import ROOT, stage_reference  # noqa: E402

# 1-D inputs: NaN, +-inf, pairs 1e200 apart (r2 overflows to +inf), a duplicated point
X1 = np.array([0.0, 0.3, np.nan, np.inf, -np.inf, 1e200, -1e200, 0.3])
X2 = np.array([0.0, 1.1, 0.3, np.nan, np.inf, -1e200, 5.0])


def kernel_zoo(kernels):
    """name -> (kernel factory, parameter-vector edits {index: value}, ndim).  The names say which device evaluator
    the kernel takes: the 1-D specialised shapes, ProfileND (one radial kernel in 2-3 dimensions) or the interpreter."""
    zoo = {}
    for sign, tag in ((1, "pos"), (-1, "neg")):
        zoo["m32_1d_logM_%s" % tag] = (lambda: 2.0 * kernels.Matern32Kernel(0.7), {1: sign * 720.0}, 1)
        zoo["m52_1d_logM_%s" % tag] = (lambda: 2.0 * kernels.Matern52Kernel(0.7), {1: sign * 720.0}, 1)
        zoo["expsq_1d_logM_%s" % tag] = (lambda: 2.0 * kernels.ExpSquaredKernel(0.7), {1: sign * 720.0}, 1)
        zoo["m32_1d_logc_%s" % tag] = (lambda: 2.0 * kernels.Matern32Kernel(0.7), {0: sign * 800.0}, 1)
        zoo["es2_gamma_%s" % tag] = (lambda: kernels.ExpSine2Kernel(gamma=1.0, log_period=0.5), {0: sign * 1e308}, 1)
        zoo["ratquad_logalpha_%s" % tag] = (lambda: kernels.RationalQuadraticKernel(log_alpha=0.3, metric=1.2),
                                           {0: sign * 700.0}, 1)
        zoo["m32_3d_iso_logM_%s" % tag] = (lambda: kernels.Matern32Kernel(0.5, ndim=3), {0: sign * 720.0}, 3)
        zoo["m52_2d_axis_logM_%s" % tag] = (lambda: kernels.Matern52Kernel([0.5, 2.0], ndim=2), {1: sign * 720.0}, 2)
    zoo["m32_1d"] = (lambda: 2.0 * kernels.Matern32Kernel(0.7), {}, 1)
    zoo["m52_1d"] = (lambda: 2.0 * kernels.Matern52Kernel(0.7), {}, 1)
    zoo["exp_1d"] = (lambda: 2.0 * kernels.ExpKernel(0.7), {}, 1)
    zoo["qp_sum_1d"] = (lambda: 1.0 * kernels.Matern32Kernel(1.0)
                        + 0.5 * kernels.ExpSine2Kernel(gamma=1.0, log_period=np.log(3.0)), {}, 1)
    zoo["m32_3d_iso"] = (lambda: kernels.Matern32Kernel(0.5, ndim=3), {}, 3)
    zoo["m52_2d_axis"] = (lambda: kernels.Matern52Kernel([0.5, 2.0], ndim=2), {}, 2)
    zoo["m32_3d_sum"] = (lambda: kernels.Matern32Kernel(0.5, ndim=3) + kernels.ExpSquaredKernel(1.0, ndim=3), {}, 3)
    return zoo


def inputs(ndim):
    """(x1, x2) with the 1-D set in the first coordinate and finite values elsewhere"""
    if ndim == 1:
        return X1[:, None].copy(), X2[:, None].copy()
    rng = np.random.default_rng(ndim)
    x1 = np.concatenate([X1[:, None], rng.normal(size=(len(X1), ndim - 1))], axis=1)
    x2 = np.concatenate([X2[:, None], rng.normal(size=(len(X2), ndim - 1))], axis=1)
    x2[1, ndim - 1] = np.nan   # a NaN in a later coordinate too
    return x1, x2


def make_kernel(zoo, name):
    mk, edits, nd = zoo[name]
    k = mk()
    v = k.get_parameter_vector(include_frozen=True)
    for i, val in edits.items():
        v[i] = val
    k.set_parameter_vector(v, include_frozen=True)
    return k, nd


# dense end-to-end problems: N points on [0, 10) with one defect each
E2E_N = 64


def e2e_problem(case):
    rng = np.random.default_rng(5)
    x = np.sort(rng.uniform(0, 10, E2E_N))
    yerr = 0.1 * np.ones(E2E_N)
    y = np.sin(x)
    kernel, vec = "m32", None
    if case == "nan_x":
        x[17] = np.nan
    elif case == "inf_x":
        x[17] = np.inf
    elif case == "nan_yerr":
        yerr[9] = np.nan
    elif case == "nan_y":
        y[40] = np.nan
    elif case in ("logM_neg", "logM_pos"):
        vec = {1: (-720.0 if case == "logM_neg" else 720.0)}
    elif case in ("logc_neg", "logc_pos"):
        vec = {0: (-800.0 if case == "logc_neg" else 800.0)}
    elif case == "dup_yerr0":
        x[20:24] = x[20]
        yerr[:] = 0.0
    elif case != "clean":
        raise ValueError(case)
    return x, yerr, y, kernel, vec


E2E_CASES = ("clean", "nan_x", "inf_x", "nan_yerr", "nan_y", "logM_neg", "logM_pos", "logc_neg", "logc_pos",
             "dup_yerr0")


def e2e_kernel(kernels, vec):
    k = 1.5 * kernels.Matern32Kernel(1.0)
    if vec:
        v = k.get_parameter_vector()
        for i, val in vec.items():
            v[i] = val
        k.set_parameter_vector(v)
    return k


def main():
    george = stage_reference()
    from george import kernels
    out = {}
    zoo = kernel_zoo(kernels)
    out["manifest__kernels"] = np.array(sorted(zoo))
    for name in sorted(zoo):
        k, nd = make_kernel(zoo, name)
        x1, x2 = inputs(nd)
        with np.errstate(all="ignore"):
            out[name + "__value"] = k.get_value(x1, x2)
            out[name + "__grad"] = k.get_gradient(x1, x2, include_frozen=True)
            out[name + "__x1grad"] = k.get_x1_gradient(x1, x2)
        out[name + "__params"] = k.get_parameter_vector(include_frozen=True)
    out["manifest__e2e"] = np.array(E2E_CASES)
    for case in E2E_CASES:
        x, yerr, y, _, vec = e2e_problem(case)
        outcome = None
        try:
            gp = george.GP(e2e_kernel(kernels, vec))
            gp.compute(x, yerr)
            ll = gp.log_likelihood(y, quiet=False)
            outcome = "finite" if np.isfinite(ll) else "-inf"
            out["e2e__%s__ll" % case] = np.array(ll)
        except Exception as exc:  # noqa: BLE001 - the class is the golden value
            outcome = type(exc).__name__
        gp = george.GP(e2e_kernel(kernels, vec))
        try:
            gp.compute(x, yerr)
        except Exception:  # noqa: BLE001 - compute may fail; log_likelihood(quiet=True) must still answer
            pass
        try:   # the reference's quiet path still raises when y itself is not finite (scipy's cho_solve checks it)
            quiet = "%r" % float(gp.log_likelihood(y, quiet=True))
        except Exception as exc:  # noqa: BLE001
            quiet = type(exc).__name__
        out["e2e__%s__quiet" % case] = np.array(quiet)
        out["e2e__%s__outcome" % case] = np.array(outcome)
    path = os.path.join(ROOT, "tests", "golden", "reference_nonfinite.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, "with", len(out), "arrays")
    for case in E2E_CASES:
        print(" ", case, out["e2e__%s__outcome" % case], out["e2e__%s__quiet" % case])


if __name__ == "__main__":
    main()
