# -*- coding: utf-8 -*-
"""GP.batch_predict on the host: the argument checks that run before any device call, the empty results, the error
raised without a device, and the per-vector loop every solver without a batched path takes."""
import numpy as np
import pytest


def _dense_gp():
    import george_b200 as george
    from george_b200 import kernels
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0))
    gp._x = np.linspace(0, 1, 5)[:, None]  # what compute() would leave, without touching the device
    gp._yerr2 = np.zeros(5)
    return gp


def test_argument_checks_run_before_any_device_call():
    import george_b200 as george
    from george_b200 import kernels
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0))
    with pytest.raises(RuntimeError, match="You need to compute the model first"):
        gp.batch_predict(np.zeros((2, len(gp))), np.zeros(3), np.zeros(4))
    gp = _dense_gp()
    for bad in (np.zeros(len(gp)), np.zeros((2, len(gp) + 1)), np.zeros((1, 2, len(gp)))):
        with pytest.raises(ValueError, match="vectors must have shape"):
            gp.batch_predict(bad, np.zeros(5), np.zeros(4))
    with pytest.raises(ValueError, match="Dimension mismatch"):
        gp.batch_predict(np.zeros((2, len(gp))), np.zeros(4), np.zeros(4))        # y's length
    with pytest.raises(ValueError, match="Dimension mismatch"):
        gp.batch_predict(np.zeros((2, len(gp))), np.zeros(5), np.zeros((4, 2)))   # t's dimension


@pytest.mark.parametrize("kw,shape", [(dict(return_cov=False), None), (dict(return_var=True), "var"),
                                      (dict(), "cov"), (dict(return_cov=True, return_var=True), "var")])
def test_empty_shapes(kw, shape):
    gp = _dense_gp()
    for nb, ns in ((0, 7), (3, 0), (0, 0)):
        got = gp.batch_predict(np.zeros((nb, len(gp))), np.zeros(5), np.zeros(ns), **kw)
        if shape is None:
            assert isinstance(got, np.ndarray) and got.shape == (nb, ns)
            continue
        mu, out = got
        assert mu.shape == (nb, ns)
        assert out.shape == ((nb, ns) if shape == "var" else (nb, ns, ns))


def test_dense_batch_without_device_raises():
    """No CPU fallback: with valid arguments and no H100, the batched dense path raises BGPError."""
    import george_b200 as george
    from george_b200 import _lib, kernels
    from george_b200._spec import flatten
    if _lib.load().bgp_device_count() > 0:
        pytest.skip("a GPU is present")
    k = 1.0 * kernels.ExpSquaredKernel(1.0)
    for what in (None, "var", "cov"):
        with pytest.raises(_lib.BGPError):
            george.BasicSolver.batch_predict(flatten(k), np.zeros((2, len(k))), np.linspace(0, 1, 5),
                                             np.ones((2, 5)), np.ones((2, 5)), np.linspace(0, 1, 3), what)
    with pytest.raises(ValueError):
        george.BasicSolver.batch_predict(flatten(k), np.zeros((2, len(k))), np.linspace(0, 1, 5),
                                         np.ones((2, 5)), np.ones((2, 5)), np.linspace(0, 1, 3), "std")
    gp = _dense_gp()
    with pytest.raises(_lib.BGPError):
        gp.batch_predict(np.zeros((2, len(gp))), np.zeros(5), np.linspace(0, 1, 3), return_var=True)
    assert george.HODLRSolver.batch_predict is None
    assert getattr(george.TrivialSolver, "batch_predict", None) is None


def _trivial_gp():
    import george_b200 as george
    gp = george.GP(mean=0.3, fit_mean=True, white_noise=np.log(0.2), fit_white_noise=True)
    assert gp.solver_type is george.TrivialSolver
    rng = np.random.default_rng(2)
    x = np.sort(rng.uniform(0, 5, 40))
    gp.compute(x, 0.05 + 0.01 * rng.uniform(size=40))
    y = np.sin(x) + 0.1 * rng.standard_normal(40)
    return gp, y


class _HostKernel(object):
    """A duck-typed numpy kernel for GP.predict's ``kernel=`` (what it calls: get_value, matvec), so that the loop
    runs without a device."""

    def get_value(self, x1, x2=None, diag=False):
        x1 = np.asarray(x1, dtype=np.float64).reshape(len(x1), -1)
        if diag:
            return np.ones(len(x1))
        x2 = x1 if x2 is None else np.asarray(x2, dtype=np.float64).reshape(len(x2), -1)
        d = x1[:, None, 0] - x2[None, :, 0]
        return np.exp(-0.5 * d * d)

    def matvec(self, x1, x2, v):
        return np.dot(self.get_value(x1, x2), v)


def test_explicit_kernel_takes_the_loop_and_restores_state():
    # (the trivial solver solves one right-hand side at a time, so only the mean of predict runs on it)
    kw = dict(return_cov=False)
    gp, y = _trivial_gp()
    gp.log_likelihood(y)
    rng = np.random.default_rng(3)
    vecs = gp.get_parameter_vector() + 0.3 * rng.standard_normal((4, len(gp)))
    t = np.linspace(0, 5, 6)
    k = _HostKernel()
    before = (gp.get_parameter_vector(include_frozen=True).copy(), gp.computed, gp.solver, gp.kernel.dirty,
              gp._alpha, gp._y, gp._const)
    got = gp.batch_predict(vecs, y, t, kernel=k, **kw)
    after = (gp.get_parameter_vector(include_frozen=True), gp.computed, gp.solver, gp.kernel.dirty, gp._alpha,
             gp._y, gp._const)
    assert np.array_equal(before[0], after[0])
    assert before[1] == after[1] and before[3] == after[3] and before[6] == after[6]
    assert before[2] is after[2] and before[4] is after[4] and before[5] is after[5]
    p0 = gp.get_parameter_vector()
    for b, v in enumerate(vecs):
        gp.set_parameter_vector(v)
        want = gp.predict(y, t, kernel=k, **kw)
        if isinstance(want, tuple):
            assert np.array_equal(got[0][b], want[0]) and np.array_equal(got[1][b], want[1])
        else:
            assert np.array_equal(got[b], want)
    gp.set_parameter_vector(p0)

    vecs[2, 0] = np.nan  # a non-finite mean: the loop's ValueError, and the GP restored
    gp.predict(y, t, kernel=k, **kw)  # (the reference loop above left the GP at another factorisation)
    solver, alpha = gp.solver, gp._alpha
    with pytest.raises(ValueError, match="mean function"):
        gp.batch_predict(vecs, y, t, kernel=k, **kw)
    assert np.array_equal(gp.get_parameter_vector(include_frozen=True), before[0])
    assert gp.solver is solver and gp._alpha is alpha and gp.computed
