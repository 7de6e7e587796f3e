# -*- coding: utf-8 -*-
"""GP.batch_log_likelihood on the host: the kernel-spec patching it relies on, the per-vector loop every solver without
a batched path takes, and the argument checks that run before any device call."""
import ctypes as C

import numpy as np
import pytest

from conftest import make_kernels, reference_kernel_list


def _all_kernels():
    zoo = [(name, k) for name, k in make_kernels()]
    zoo += [("ref{0}".format(i), k) for i, k in enumerate(reference_kernel_list())]
    return zoo


def test_patched_specs_equal_flatten_after_set_parameter_vector():
    from george_b200._spec import KernelSpec, flatten, num_params, patch_specs
    rng = np.random.default_rng(1)
    for name, k in _all_kernels():
        template = flatten(k)
        p0 = k.get_parameter_vector(include_frozen=True)
        assert num_params(template) == len(p0), name
        params = p0 + 0.1 * rng.standard_normal((3, len(p0)))
        patched = patch_specs(template, params)
        try:
            for b in range(3):
                k.set_parameter_vector(params[b], include_frozen=True)
                ref = flatten(k)
                assert C.string_at(C.byref(patched[b]), C.sizeof(KernelSpec)) == \
                    C.string_at(C.byref(ref), C.sizeof(KernelSpec)), (name, b)
        finally:
            k.set_parameter_vector(p0, include_frozen=True)
    with pytest.raises(ValueError):
        patch_specs(template, np.zeros((2, len(p0) + 1)))


def _trivial_gp():
    import george_b200 as george
    gp = george.GP(mean=0.3, fit_mean=True, white_noise=np.log(0.2), fit_white_noise=True)
    assert gp.solver_type is george.TrivialSolver
    rng = np.random.default_rng(2)
    x = np.sort(rng.uniform(0, 5, 40))
    gp.compute(x, 0.05 + 0.01 * rng.uniform(size=40))
    y = np.sin(x) + 0.1 * rng.standard_normal(40)
    return gp, y


def test_trivial_solver_batch_equals_loop_and_restores_state():
    gp, y = _trivial_gp()
    gp.log_likelihood(y)
    rng = np.random.default_rng(3)
    vecs = gp.get_parameter_vector() + 0.3 * rng.standard_normal((6, len(gp)))
    vecs[2, 0] = np.nan  # a non-finite mean: -inf under quiet
    before = (gp.get_parameter_vector(include_frozen=True).copy(), gp.computed, gp.solver, gp.kernel.dirty, gp._alpha)
    got = gp.batch_log_likelihood(vecs, y, quiet=True)
    after = (gp.get_parameter_vector(include_frozen=True), gp.computed, gp.solver, gp.kernel.dirty, gp._alpha)
    assert np.array_equal(before[0], after[0]) and before[1:] == after[1:]

    want = np.empty(len(vecs))
    p0 = gp.get_parameter_vector()
    for b, v in enumerate(vecs):
        gp.set_parameter_vector(v)
        want[b] = gp.log_likelihood(y, quiet=True)
    gp.set_parameter_vector(p0)
    assert np.isneginf(got[2])
    assert np.array_equal(got, want)

    with pytest.raises(ValueError, match="mean function"):
        gp.batch_log_likelihood(vecs, y, quiet=False)
    assert np.array_equal(gp.get_parameter_vector(include_frozen=True), before[0])


def test_argument_checks_run_before_any_device_call():
    import george_b200 as george
    from george_b200 import kernels
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0))
    with pytest.raises(RuntimeError, match="You need to compute the model first"):
        gp.batch_log_likelihood(np.zeros((2, len(gp))), np.zeros(3))
    gp._x = np.linspace(0, 1, 5)[:, None]  # what compute() would leave, without touching the device
    gp._yerr2 = np.zeros(5)
    for bad in (np.zeros(len(gp)), np.zeros((2, len(gp) + 1)), np.zeros((1, 2, len(gp)))):
        with pytest.raises(ValueError):
            gp.batch_log_likelihood(bad, np.zeros(5))
    assert gp.batch_log_likelihood(np.zeros((0, len(gp))), np.zeros(5)).shape == (0,)


def test_dense_batch_without_device_raises():
    """No CPU fallback: with valid arguments and no H100, the batched dense path raises BGPError."""
    import george_b200 as george
    from george_b200 import _lib, kernels
    from george_b200._spec import flatten
    if _lib.load().bgp_device_count() > 0:
        pytest.skip("a GPU is present")
    k = 1.0 * kernels.ExpSquaredKernel(1.0)
    with pytest.raises(_lib.BGPError):
        george.BasicSolver.batch_log_likelihood(flatten(k), np.zeros((2, len(k))), np.linspace(0, 1, 5),
                                                np.ones((2, 5)), np.ones((2, 5)))
    gp = george.GP(k)
    gp._x = np.linspace(0, 1, 5)[:, None]
    gp._yerr2 = np.zeros(5)
    with pytest.raises(_lib.BGPError):
        gp.batch_log_likelihood(np.zeros((2, len(gp))), np.zeros(5))
    assert george.HODLRSolver.batch_log_likelihood is None
    assert getattr(george.TrivialSolver, "batch_log_likelihood", None) is None
