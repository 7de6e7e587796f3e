# -*- coding: utf-8 -*-
"""GP.batch_grad_predict on the host: the argument checks that run before any device call (order, types, messages),
the empty results, the error raised without a device, and the per-vector loop that solvers without a batched path and
an explicit kernel take."""
import numpy as np
import pytest


def _dense_gp(kernel=None, n=5):
    import george_b200 as george
    from george_b200 import kernels
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0) if kernel is None else kernel)
    nd = gp.kernel.ndim
    gp._x = np.linspace(0, 1, n * nd).reshape(n, nd)  # what compute() would leave, without touching the device
    gp._yerr2 = np.zeros(n)
    return gp


class _NoDevice(object):
    """Replaces the batched solver hook: any call means device work started before an argument check."""

    def __call__(self, *args, **kwargs):
        raise AssertionError("the device was reached")


def test_argument_checks_run_in_order_before_any_device_call(monkeypatch):
    import george_b200 as george
    from george_b200 import kernels
    from george_b200.modeling import Model
    monkeypatch.setattr(george.BasicSolver, "batch_predict_grad", _NoDevice())

    class LineModel(Model):
        parameter_names = ("m",)

        def get_value(self, t):
            return self.m * t.flatten()

    # 1. a non-constant mean, before the computed check
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0), mean=LineModel(m=0.5))
    with pytest.raises(NotImplementedError, match="only a constant mean is supported"):
        gp.batch_grad_predict(np.zeros((2, len(gp))), np.zeros(3), np.zeros(4))
    # 2. not computed, before the shape of vectors
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0))
    with pytest.raises(RuntimeError, match="You need to compute the model first"):
        gp.batch_grad_predict(np.zeros(3), np.zeros(3), np.zeros((4, 2)))
    gp = _dense_gp()
    # 3. the shape of vectors, before y's length
    for bad in (np.zeros(len(gp)), np.zeros((2, len(gp) + 1)), np.zeros((1, 2, len(gp)))):
        with pytest.raises(ValueError, match="vectors must have shape"):
            gp.batch_grad_predict(bad, np.zeros(4), np.zeros((4, 2)))
    # 4. y's length, before t's dimension
    with pytest.raises(ValueError, match="^Dimension mismatch$"):
        gp.batch_grad_predict(np.zeros((2, len(gp))), np.zeros(4), np.zeros((4, 2)))
    # 5. t's dimension
    with pytest.raises(ValueError, match="^Dimension mismatch$"):
        gp.batch_grad_predict(np.zeros((2, len(gp))), np.zeros(5), np.zeros((4, 2)))
    # 6. more than 8 input dimensions
    gp9 = _dense_gp(1.0 * kernels.ExpSquaredKernel(1.0, ndim=9, axes=[0, 1, 2]))
    with pytest.raises(ValueError, match=r"at most 8 dimensions \(got 9\)"):
        gp9.batch_grad_predict(np.zeros((2, len(gp9))), np.zeros(5), np.zeros((4, 9)))
    with pytest.raises(ValueError, match=r"at most 8 dimensions \(got 9\)"):
        gp9.batch_grad_predict(np.zeros((0, len(gp9))), np.zeros(5), np.zeros((0, 9)))


def test_checks_match_grad_predict_messages():
    """The member-independent checks raise what grad_predict / batch_predict raise for the same arguments."""
    gp = _dense_gp()
    for y, t in ((np.zeros(4), np.zeros(3)), (np.zeros(5), np.zeros((3, 2)))):
        with pytest.raises(ValueError) as a:
            gp.batch_grad_predict(np.zeros((1, len(gp))), y, t)
        with pytest.raises(ValueError) as b:
            gp.batch_predict(np.zeros((1, len(gp))), y, t)
        assert str(a.value) == str(b.value)


@pytest.mark.parametrize("return_var", [False, True])
def test_empty_shapes(monkeypatch, return_var):
    import george_b200 as george
    from george_b200 import kernels
    monkeypatch.setattr(george.BasicSolver, "batch_predict_grad", _NoDevice())
    for kernel, nd in ((None, 1), (1.0 * kernels.Matern52Kernel(1.0, ndim=3), 3)):
        gp = _dense_gp(kernel)
        for nb, ns in ((0, 7), (3, 0), (0, 0)):
            t = np.zeros(ns) if nd == 1 else np.zeros((ns, nd))
            got = gp.batch_grad_predict(np.zeros((nb, len(gp))), np.zeros(5), t, return_var=return_var)
            assert len(got) == (4 if return_var else 2)
            assert got[0].shape == (nb, ns) and got[-1].shape == (nb, ns, nd)
            if return_var:
                assert got[1].shape == (nb, ns) and got[2].shape == (nb, ns, nd)
            assert all(a.dtype == np.float64 for a in got)


def test_dense_batch_without_device_raises():
    """No CPU fallback: with valid arguments and no H100, the batched dense path raises BGPError."""
    import george_b200 as george
    from george_b200 import _lib, kernels
    from george_b200._spec import flatten
    if _lib.load().bgp_device_count() > 0:
        pytest.skip("a GPU is present")
    k = 1.0 * kernels.ExpSquaredKernel(1.0)
    for rv in (False, True):
        with pytest.raises(_lib.BGPError):
            george.BasicSolver.batch_predict_grad(flatten(k), np.zeros((2, len(k))), np.linspace(0, 1, 5),
                                                  np.ones((2, 5)), np.ones((2, 5)), np.linspace(0, 1, 3), rv)
    with pytest.raises(ValueError, match="yerr and r must have shape"):
        george.BasicSolver.batch_predict_grad(flatten(k), np.zeros((2, len(k))), np.linspace(0, 1, 5),
                                              np.ones((3, 5)), np.ones((2, 5)), np.linspace(0, 1, 3), False)
    gp = _dense_gp()
    with pytest.raises(_lib.BGPError):
        gp.batch_grad_predict(np.zeros((2, len(gp))), np.zeros(5), np.linspace(0, 1, 3), return_var=True)
    assert george.HODLRSolver.batch_predict_grad is None
    assert getattr(george.TrivialSolver, "batch_predict_grad", None) is None


def test_abi_rejects_wide_inputs_before_any_work():
    from george_b200 import _lib, kernels
    from george_b200._spec import flatten
    import ctypes as C
    lib = _lib.load()
    k = kernels.ExpSquaredKernel(1.0, ndim=9, axes=[0, 1, 2])
    h = C.c_void_p()
    _lib.check(lib.bgp_dense_batch_create(C.byref(h)))
    try:
        spec = flatten(k)
        x = np.zeros((4, 9))
        arr = np.zeros(64)
        info = np.zeros(2, dtype=np.int32)
        st = lib.bgp_dense_batch_predict_grad(h, C.byref(spec), _lib.ptr(arr), 2, len(k), _lib.ptr(x), 4, 9,
                                              _lib.ptr(arr), _lib.ptr(arr), _lib.ptr(x), 4, 1, _lib.ptr(arr),
                                              _lib.ptr(arr), _lib.ptr(arr), _lib.ptr(arr), _lib.ptr(info))
        assert st == _lib.BGP_ERR_INVALID
        assert "at most 8 dimensions" in lib.bgp_last_error().decode()
    finally:
        lib.bgp_dense_batch_destroy(h)


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
    """A duck-typed numpy kernel for GP.grad_predict's ``kernel=`` (what it calls: matvec and
    kernel.x1_gradient_matvec), so that the loop runs without a device: k(a, b) = exp(-(a - b)^2 / 2) in 1-D."""

    def __init__(self):
        self.kernel = self

    def get_value(self, x1, x2=None, diag=False):
        x1 = np.asarray(x1, dtype=np.float64).reshape(len(x1), -1)
        if diag:
            return np.ones(len(x1))
        x2 = x1 if x2 is None else np.asarray(x2, dtype=np.float64).reshape(len(x2), -1)
        d = x1[:, None, 0] - x2[None, :, 0]
        return np.exp(-0.5 * d * d)

    def matvec(self, x1, x2, v):
        return np.dot(self.get_value(x1, x2), v)

    def x1_gradient_matvec(self, x1, x2, v, scale=1.0, add_prior=False):
        x1 = np.asarray(x1, dtype=np.float64).reshape(len(x1), -1)
        x2 = np.asarray(x2, dtype=np.float64).reshape(len(x2), -1)
        d = x1[:, None, 0] - x2[None, :, 0]
        g = -d * np.exp(-0.5 * d * d)
        return scale * np.dot(g, v)[:, None]


def _state(gp):
    return (gp.get_parameter_vector(include_frozen=True).copy(), gp.computed, gp.solver, gp._alpha, gp._y,
            gp._const, [m.dirty for m in gp.models.values()])


def _assert_state(gp, st):
    now = _state(gp)
    assert np.array_equal(st[0], now[0])
    assert now[1] == st[1] and now[5] == st[5] and now[6] == st[6]
    assert now[2] is st[2] and now[3] is st[3] and now[4] is st[4]


def test_trivial_solver_and_explicit_kernel_take_the_loop_and_restore_state():
    gp, y = _trivial_gp()
    gp.log_likelihood(y)
    k = _HostKernel()
    gp.predict(y, np.zeros(1), return_cov=False, kernel=k)  # a cached solve to restore
    rng = np.random.default_rng(3)
    vecs = gp.get_parameter_vector() + 0.3 * rng.standard_normal((4, len(gp)))
    t = np.linspace(0, 5, 6)
    st = _state(gp)
    mu, dmu = gp.batch_grad_predict(vecs, y, t, kernel=k)
    _assert_state(gp, st)
    assert mu.shape == (4, 6) and dmu.shape == (4, 6, 1)
    p0 = gp.get_parameter_vector()
    for b, v in enumerate(vecs):
        gp.set_parameter_vector(v)
        m1, d1 = gp.grad_predict(y, t, kernel=k)
        assert np.array_equal(mu[b], m1) and np.array_equal(dmu[b], d1)
    gp.set_parameter_vector(p0)

    # the trivial solver without a kernel: its loop reaches the device, so only the route is checked here
    assert getattr(type(gp.solver), "batch_predict_grad", None) is None

    vecs[2, 0] = np.nan  # a non-finite mean: the loop's ValueError, and the GP restored
    gp.log_likelihood(y)
    st = _state(gp)
    with pytest.raises(ValueError, match="mean function"):
        gp.batch_grad_predict(vecs, y, t, kernel=k)
    _assert_state(gp, st)
