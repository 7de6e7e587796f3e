# -*- coding: utf-8 -*-
"""GP.batch_grad_log_likelihood on the host: the argument checks that run before any device call, the empty results,
the error raised without a device, and the per-vector loop every solver without a batched path takes."""
import numpy as np
import pytest


def _dense_gp():
    import george_b200 as george
    from george_b200 import kernels
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0), white_noise=np.log(0.1), fit_white_noise=True)
    gp._x = np.linspace(0, 1, 5)[:, None]  # what compute() would leave, without touching the device
    gp._yerr2 = np.zeros(5)
    return gp


def test_argument_checks_run_before_any_device_call():
    import george_b200 as george
    from george_b200 import kernels
    from george_b200._spec import flatten
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0))
    with pytest.raises(RuntimeError, match="You need to compute the model first"):
        gp.batch_grad_log_likelihood(np.zeros((2, len(gp))), np.zeros(3))
    gp = _dense_gp()
    for bad in (np.zeros(len(gp)), np.zeros((2, len(gp) + 1)), np.zeros((1, 2, len(gp)))):
        with pytest.raises(ValueError, match="vectors must have shape"):
            gp.batch_grad_log_likelihood(bad, np.zeros(5))
    for quiet in (False, True):
        with pytest.raises(ValueError, match="Dimension mismatch"):
            gp.batch_grad_log_likelihood(np.zeros((2, len(gp))), np.zeros(4), quiet=quiet)   # y's length

    k = 1.0 * kernels.ExpSquaredKernel(1.0)
    spec, x, ones = flatten(k), np.linspace(0, 1, 5), np.ones((2, 5))
    which = np.ones(len(k), dtype=np.uint32)
    fn = george.BasicSolver.batch_grad_terms
    with pytest.raises(ValueError, match="params must have shape"):
        fn(spec, np.zeros((2, len(k) + 1)), x, ones, ones, which)
    with pytest.raises(ValueError, match="yerr and r must have shape"):
        fn(spec, np.zeros((2, len(k))), x, np.ones((3, 5)), ones, which)
    with pytest.raises(ValueError, match="which must have shape"):
        fn(spec, np.zeros((2, len(k))), x, ones, ones, which[:1])
    with pytest.raises(ValueError, match="x must have shape"):
        fn(spec, np.zeros((2, len(k))), np.zeros((0, 1)), np.ones((2, 0)), np.ones((2, 0)), which)
    with pytest.raises(RuntimeError, match="dimension mismatch"):
        fn(spec, np.zeros((2, len(k))), np.zeros((5, 2)), ones, ones, which)


def test_more_than_64_parameters_are_rejected_before_any_device_call():
    import george_b200 as george
    from george_b200 import kernels
    from george_b200._spec import flatten
    k = 1.0 * kernels.ExpSquaredKernel(np.eye(8), ndim=8)
    for _ in range(2):
        k = k + 1.0 * kernels.ExpSquaredKernel(np.eye(8), ndim=8)
    assert k.full_size > 64
    p = np.tile(k.get_parameter_vector(include_frozen=True), (2, 1))
    with pytest.raises(ValueError, match="64"):
        george.BasicSolver.batch_grad_terms(flatten(k), p, np.zeros((5, 8)), np.ones((2, 5)), np.ones((2, 5)),
                                            np.ones(k.full_size, dtype=np.uint32))


def test_empty_batch():
    gp = _dense_gp()
    grad = gp.batch_grad_log_likelihood(np.zeros((0, len(gp))), np.zeros(5))
    assert grad.shape == (0, len(gp))
    ll, grad = gp.batch_grad_log_likelihood(np.zeros((0, len(gp))), np.zeros(5), return_log_likelihood=True)
    assert ll.shape == (0,) and grad.shape == (0, len(gp))
    from george_b200 import BasicSolver, kernels
    from george_b200._spec import flatten
    k = 1.0 * kernels.ExpSquaredKernel(1.0)
    out = BasicSolver.batch_grad_terms(flatten(k), np.zeros((0, len(k))), np.linspace(0, 1, 5), np.ones((0, 5)),
                                       np.ones((0, 5)), np.ones(len(k), dtype=np.uint32))
    assert [a.shape for a in out] == [(0,), (0,), (0, 5), (0, len(k)), (0, 5), (0,)]


def test_dense_batch_without_device_raises():
    """No CPU fallback: with valid arguments and no H100, the batched dense path raises BGPError."""
    import george_b200 as george
    from george_b200 import _lib, kernels
    from george_b200._spec import flatten
    if _lib.load().bgp_device_count() > 0:
        pytest.skip("a GPU is present")
    k = 1.0 * kernels.ExpSquaredKernel(1.0)
    with pytest.raises(_lib.BGPError):
        george.BasicSolver.batch_grad_terms(flatten(k), np.zeros((2, len(k))), np.linspace(0, 1, 5),
                                            np.ones((2, 5)), np.ones((2, 5)), np.ones(len(k), dtype=np.uint32))
    gp = _dense_gp()
    with pytest.raises(_lib.BGPError):
        gp.batch_grad_log_likelihood(np.zeros((2, len(gp))), np.zeros(5))
    assert george.HODLRSolver.batch_grad_terms is None
    assert getattr(george.TrivialSolver, "batch_grad_terms", None) is None


def _trivial_gp():
    import george_b200 as george
    gp = george.GP(mean=0.3, fit_mean=True, white_noise=np.log(0.2))
    assert gp.solver_type is george.TrivialSolver
    rng = np.random.default_rng(2)
    x = np.sort(rng.uniform(0, 5, 40))
    gp.compute(x, 0.05 + 0.01 * rng.uniform(size=40))
    y = np.sin(x) + 0.1 * rng.standard_normal(40)
    return gp, y


def _loop(gp, vecs, y, quiet, return_ll):
    p0 = gp.get_parameter_vector()
    ll, grad = np.empty(len(vecs)), np.empty((len(vecs), len(gp)))
    for b, v in enumerate(vecs):
        gp.set_parameter_vector(v)
        if return_ll:
            ll[b] = gp.log_likelihood(y, quiet=quiet)
        grad[b] = gp.grad_log_likelihood(y, quiet=quiet)
    gp.set_parameter_vector(p0)
    return (ll, grad) if return_ll else grad


def _state(gp):
    return (gp.get_parameter_vector(include_frozen=True).copy(), gp.computed, gp.solver, gp._alpha, gp._y, gp._const,
            [m.dirty for m in gp.models.values()])


def _assert_state(gp, st):
    now = _state(gp)
    assert np.array_equal(st[0], now[0])
    assert now[1] == st[1] and now[5] == st[5] and now[6] == st[6]
    assert now[2] is st[2] and now[3] is st[3] and now[4] is st[4]


def test_trivial_solver_takes_the_loop_and_restores_state():
    gp, y = _trivial_gp()
    gp.log_likelihood(y)
    rng = np.random.default_rng(3)
    vecs = gp.get_parameter_vector() + 0.3 * rng.standard_normal((4, len(gp)))
    for return_ll in (False, True):
        st = _state(gp)
        got = gp.batch_grad_log_likelihood(vecs, y, return_log_likelihood=return_ll)
        _assert_state(gp, st)
        want = _loop(gp, vecs, y, False, return_ll)
        if return_ll:
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
        else:
            assert np.array_equal(got, want)
        gp.log_likelihood(y)  # (the reference loop above left the GP at another factorisation)

    vecs[2, 0] = np.nan  # a non-finite mean: -inf and a zero gradient under quiet, the loop's ValueError otherwise
    st = _state(gp)
    ll, grad = gp.batch_grad_log_likelihood(vecs, y, quiet=True, return_log_likelihood=True)
    _assert_state(gp, st)
    assert np.isneginf(ll[2]) and np.all(grad[2] == 0.0)
    want = _loop(gp, vecs, y, True, True)
    assert np.array_equal(ll, want[0]) and np.array_equal(grad, want[1])
    gp.log_likelihood(y)
    st = _state(gp)
    with pytest.raises(ValueError, match="mean function"):
        gp.batch_grad_log_likelihood(vecs, y)
    _assert_state(gp, st)
