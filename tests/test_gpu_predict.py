# -*- coding: utf-8 -*-
"""GP.predict's variance and covariance on the device (``bgp_dense_predict`` / ``bgp_hodlr_predict``, csrc/dense.cu,
csrc/hodlr.cu, csrc/kmat_ops.cu) against an extended-precision reference and against the reference's host route
(``GP._predict_host``: K(x*, x) on the host, ``solver.apply_inverse`` on its transpose).

Errors are measured on the scale of the prior, ``max|out - ref| / max|K**|``: ``var = k** - q`` cancels near the data,
so an error relative to the result itself says nothing about the computation.
"""
import ctypes as C
import pickle

import numpy as np
import pytest

import hiprec

pytestmark = pytest.mark.gpu

LD = np.longdouble

# bars: 10-60x the largest value measured on one H100 80GB HBM3 (SXM, 400 W power limit)
EXACT_TOL = 1e-13        # dense vs the longdouble reference                                   (measured 2.5e-15)
HODLR_EXACT_TOL = 5e-12  # exact-K HODLR vs the longdouble reference, cond(K) ~ 1e4            (measured 1.3e-13)
HOST_TOL = 1e-13         # device vs the host path on the same factorisation                   (measured 5.3e-15)
STREAM_TOL = 1e-14       # ns = 4096 variance vs the host path at 64 of its points             (measured 3.3e-16)
CHUNK_TOL = 1e-13        # BGP_PREDICT_CHUNK=64 vs the default chunking                        (measured 4.3e-15)

DENSE_N = [1, 63, 64, 65, 700]
NS = [1, 7, 8, 9, 64, 65, 300]
CHUNKS = [None, "64", "ob64"]


@pytest.fixture
def env(monkeypatch):
    for var in ("BGP_PREDICT_CHUNK", "BGP_DENSE_OB"):
        monkeypatch.delenv(var, raising=False)
    return monkeypatch


def _set_chunking(env, mode):
    if mode == "64":
        env.setenv("BGP_PREDICT_CHUNK", "64")
    elif mode == "ob64":
        env.setenv("BGP_DENSE_OB", "64")
        env.setenv("BGP_PREDICT_CHUNK", "7")  # dense: chunks of 7 (few-RHS solves) with a ragged tail


def _err(out, ref, kss):
    return float(np.max(np.abs(np.asarray(out, dtype=LD) - np.asarray(ref, dtype=LD))) / np.max(np.abs(kss)))


def _ref_ld(kernel, L, x, xs):
    """var and cov in longdouble from the device-built K(x*, x) and K**: W = L^-1 K(x, x*), var = k** - ||W_j||^2."""
    Kxs = kernel.get_value(xs, x)
    Kss = kernel.get_value(xs)
    kd = kernel.get_value(xs, diag=True)
    n = L.shape[0]
    W = np.array(Kxs.T, dtype=LD)
    for i in range(n):
        W[i] = (W[i] - L[i, :i] @ W[:i]) / L[i, i]
    return kd.astype(LD) - np.sum(W * W, axis=0), Kss.astype(LD) - W.T @ W, Kss


_DENSE = {}


def _dense_problem(n):
    if n not in _DENSE:
        from george_b200 import kernels as K
        rng = np.random.default_rng(100 + n)
        kernel = 1.3 * K.ExpSquaredKernel(0.8)
        x = np.sort(rng.uniform(0, max(n, 2) / 40.0, n))[:, None]
        yerr = 0.2 + 0.1 * rng.uniform(size=n)
        xs = np.sort(rng.uniform(-0.5, max(n, 2) / 40.0 + 0.5, max(NS)))[:, None]
        K = kernel.get_value(x)
        K[np.diag_indices(n)] += yerr ** 2
        L = hiprec.chol_ld(K)
        var, cov, kss = _ref_ld(kernel, L, x, xs)
        _DENSE[n] = (kernel, x, yerr, xs, var, cov, kss)
    return _DENSE[n]


@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("n", DENSE_N)
def test_dense_against_extended_precision(gpu, env, record_property, n, chunk):
    import george_b200 as george
    kernel, x, yerr, xs, var_ref, cov_ref, kss = _dense_problem(n)
    _set_chunking(env, chunk)
    s = george.BasicSolver(kernel)
    s.compute(x, yerr)
    worst = 0.0
    for ns in NS:
        var = s.predictive(kernel, xs[:ns], "var")
        cov = s.predictive(kernel, xs[:ns], "cov")
        assert var.shape == (ns,) and cov.shape == (ns, ns)
        assert np.array_equal(cov, cov.T)  # lower triangle mirrored: exactly symmetric
        k = kss[:ns, :ns]
        worst = max(worst, _err(var, var_ref[:ns], k), _err(cov, cov_ref[:ns, :ns], k))
    record_property("max_err", worst)
    assert worst <= EXACT_TOL, worst


_HODLR = {}


def _exp_problem(n):
    """ExpKernel on sorted 1-D inputs is exactly rank 1 between the halves of every node: under exhaust="dense" the
    HODLR matrix is K itself (tests/test_gpu_hodlr_sweeps.py)."""
    if n not in _HODLR:
        from george_b200 import kernels as K
        rng = np.random.default_rng(7 + n)
        kernel = 1.0 * K.ExpKernel(1.0)
        x = np.sort(rng.uniform(0, n / 50.0, n))[:, None]
        yerr = 0.1 * np.ones(n)
        xs = rng.uniform(-0.5, n / 50.0 + 0.5, max(NS))[:, None]
        K = kernel.get_value(x)
        K[np.diag_indices(n)] += yerr ** 2
        L = hiprec.chol_ld(K)
        var, cov, kss = _ref_ld(kernel, L, x, xs)
        _HODLR[n] = (kernel, x, yerr, xs, var, cov, kss)
    return _HODLR[n]


@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("rng_mode", ["pernode", "reference"])
@pytest.mark.parametrize("n,min_size", [(65, 16), (300, 32), (800, 50)])
def test_hodlr_exact_k_against_extended_precision(gpu, env, record_property, n, min_size, rng_mode, chunk):
    import george_b200 as george
    kernel, x, yerr, xs, var_ref, cov_ref, kss = _exp_problem(n)
    _set_chunking(env, chunk)
    s = george.HODLRSolver(kernel, min_size=min_size, tol=1e-12, rng_mode=rng_mode, exhaust="dense")
    s.compute(x, yerr)
    worst = 0.0
    for ns in NS:
        var = s.predictive(kernel, xs[:ns], "var")
        cov = s.predictive(kernel, xs[:ns], "cov")
        assert var.shape == (ns,) and cov.shape == (ns, ns)
        k = kss[:ns, :ns]
        worst = max(worst, _err(var, var_ref[:ns], k), _err(cov, cov_ref[:ns, :ns], k))
    record_property("max_err", worst)
    assert worst <= HODLR_EXACT_TOL, worst


# ---- agreement with the host path ---------------------------------------------------------------------------------
def _points(ndim, n, rng):
    x = rng.uniform(-1.5, 1.5, (n, ndim))
    return x[np.argsort(x[:, 0])]


def _host(gp, y, xs, return_var, kernel=None):
    alpha = gp._compute_alpha(y, True)
    return gp._predict_host(alpha, gp.parse_samples(xs), return_var, gp.kernel if kernel is None else kernel)


def _check_against_host(gp, y, t, kernel=None, tol=HOST_TOL):
    """predict's var and cov (device) against GP._predict_host; returns the largest error on the prior's scale."""
    xs = gp.parse_samples(t)
    k = gp.kernel if kernel is None else kernel
    kss = k.get_value(xs)
    mu_v, var = gp.predict(y, t, return_var=True, kernel=kernel)
    mu_c, cov = gp.predict(y, t, kernel=kernel)
    mu_h, var_h = _host(gp, y, t, True, kernel)
    _, cov_h = _host(gp, y, t, False, kernel)
    assert var.shape == var_h.shape and cov.shape == cov_h.shape
    assert var.dtype == var_h.dtype == cov.dtype == cov_h.dtype == np.float64
    scale = max(np.max(np.abs(mu_h)), 1e-300)
    assert np.max(np.abs(mu_v - mu_h)) <= 1e-10 * scale and np.array_equal(mu_v, mu_c)
    err = max(_err(var, var_h, kss), _err(cov, cov_h, kss))
    assert err <= tol, err
    return err


def _zoo():
    from conftest import make_kernels
    from george_b200 import kernels as K
    zoo = list(make_kernels())
    zoo.append(("cauchy_2d", 0.7 * K.CauchyKernel(1.3, ndim=2)
                + K.DampedCosineKernel(log_period=0.1, log_decay=0.7, ndim=2, axes=[0, 1])))
    zoo.append(("damped_cos_1d", 1.0 * K.CauchyKernel(metric=1.0)
                + 0.5 * K.DampedCosineKernel(log_period=np.log(3.0), log_decay=np.log(20.0))))
    return zoo


SOLVERS = [("basic", {}), ("hodlr", {"tol": 1e-10, "min_size": 40}), ("hodlr_tol01", {"min_size": 40})]


def _make_gp(solver_name, kernel, **gp_kw):
    import george_b200 as george
    name, kw = dict((s[0], s) for s in SOLVERS)[solver_name]
    solver = george.BasicSolver if name == "basic" else george.HODLRSolver
    return george.GP(kernel, solver=solver, **dict(kw, **gp_kw))


@pytest.mark.parametrize("solver_name", [s[0] for s in SOLVERS])
@pytest.mark.parametrize("idx", range(16))
def test_kernels_against_host_path(gpu, env, record_property, idx, solver_name):
    name, kernel = _zoo()[idx]
    rng = np.random.default_rng(300 + idx)
    x = _points(kernel.ndim, 257, rng)
    y = np.sin(3 * x[:, 0])
    t = _points(kernel.ndim, 70, rng)
    gp = _make_gp(solver_name, kernel)
    gp.compute(x if kernel.ndim > 1 else x[:, 0], 0.3)
    record_property("max_err", _check_against_host(gp, y, t if kernel.ndim > 1 else t[:, 0]))


@pytest.mark.parametrize("solver_name", [s[0] for s in SOLVERS])
def test_mean_model_white_noise_and_kernel_override(gpu, env, record_property, solver_name):
    from george_b200 import kernels as K
    from george_b200.modeling import Model

    class Line(Model):
        parameter_names = ("m", "b")

        def get_value(self, x):
            return self.m * x + self.b

    rng = np.random.default_rng(11)
    x = np.sort(rng.uniform(0, 10, 400))
    y = 0.3 * x + np.sin(x) + 0.1 * rng.normal(size=x.size)
    k1 = 1.5 * K.Matern32Kernel(2.0)
    k2 = 0.4 * K.ExpSine2Kernel(gamma=2.0, log_period=np.log(3.0))
    gp = _make_gp(solver_name, k1 + k2, mean=Line(m=0.3, b=0.1), fit_mean=True, white_noise=np.log(0.05),
                  fit_white_noise=True)
    gp.compute(x, 0.1)
    t = np.linspace(-1, 11, 90)
    errs = [_check_against_host(gp, y, t), _check_against_host(gp, y, t, kernel=k1),
            _check_against_host(gp, y, t[:, None])]
    mu, var = gp.predict(y, t[:1], return_var=True)   # one test point, 1-D and 2-D t
    _, cov = gp.predict(y, t[:1, None])
    assert mu.shape == var.shape == (1,) and cov.shape == (1, 1)
    record_property("max_err", max(errs))


# ---- size and streaming -------------------------------------------------------------------------------------------
_BIG = {}


def _headline_gp():
    """Matern-3/2, N = 2^18, leaf 256, tol 1e-10, exhaust="lowrank": the headline HODLR configuration."""
    if "gp" not in _BIG:
        import george_b200 as george
        from george_b200 import kernels as K
        rng = np.random.default_rng(2024)
        n = 1 << 18
        x = np.sort(rng.uniform(0, 2000, n))
        y = np.sin(x) + 0.1 * rng.normal(size=n)
        gp = george.GP(1.0 * K.Matern32Kernel(4.0), solver=george.HODLRSolver, min_size=256, tol=1e-10,
                       exhaust="lowrank")
        gp.compute(x, 0.1)
        _BIG["gp"] = (gp, x, y, rng)
    return _BIG["gp"]


def test_headline_hodlr_against_host_path(gpu, env, record_property):
    gp, x, y, rng = _headline_gp()
    t = np.sort(rng.uniform(-5, 2005, 64))
    record_property("max_err", _check_against_host(gp, y, t))


def test_headline_hodlr_4096_variance_streams(gpu, env, record_property):
    """ns = 4096: the host path would hold ~17 GB of (N, ns) arrays.  64 random points are checked against the host
    path evaluated at those points alone; the chunk boundaries differ, so only the reduction order moves."""
    gp, x, y, rng = _headline_gp()
    t = rng.uniform(-5, 2005, 4096)
    _, var = gp.predict(y, t, return_var=True)
    assert var.shape == (4096,)
    pick = rng.choice(4096, 64, replace=False)
    _, var_h = _host(gp, y, t[pick], True)
    kd = gp.kernel.get_value(t[pick][:, None], diag=True)
    err = float(np.max(np.abs(var[pick] - var_h)) / np.max(np.abs(kd)))
    record_property("max_err", err)
    assert err <= STREAM_TOL, err


@pytest.mark.parametrize("n", [2047, 4161])
def test_dense_sizes_against_host_path(gpu, env, record_property, n):
    from george_b200 import kernels as K
    rng = np.random.default_rng(n)
    x = _points(3, n, rng)
    gp = _make_gp("basic", 1.0 * K.Matern52Kernel(0.5, ndim=3))
    gp.compute(x, 0.2)
    record_property("max_err", _check_against_host(gp, np.sin(x[:, 0] * 3), _points(3, 1000, rng)))


@pytest.mark.parametrize("solver_name", ["basic", "hodlr"])
def test_forced_chunks_match_default_chunking(gpu, env, record_property, solver_name):
    from george_b200 import kernels as K
    rng = np.random.default_rng(5)
    x = np.sort(rng.uniform(0, 30, 3000))
    gp = _make_gp(solver_name, 1.0 * K.Matern32Kernel(1.5))
    gp.compute(x, 0.1)
    y = np.sin(x)
    t = rng.uniform(-1, 31, 1000)
    kss = gp.kernel.get_value(t[:, None])
    _, var0 = gp.predict(y, t, return_var=True)
    _, cov0 = gp.predict(y, t)
    env.setenv("BGP_PREDICT_CHUNK", "64")
    _, var1 = gp.predict(y, t, return_var=True)
    _, cov1 = gp.predict(y, t)
    err = max(_err(var1, var0, kss), _err(cov1, cov0, kss))
    record_property("max_err", err)
    assert err <= CHUNK_TOL, err


# ---- determinism, edges and errors --------------------------------------------------------------------------------
@pytest.mark.parametrize("solver_name,n", [("basic", 5000), ("hodlr", 1000)])
def test_identical_calls_are_bit_identical(gpu, env, solver_name, n):
    """The reductions add in a fixed order.  The HODLR solve itself (which apply_inverse runs too) accumulates a
    node's Gram product with atomics once a half has more than 512 rows (gram_tn_kernel, csrc/hodlr_kernels.cuh), so
    its bits are reproducible only below N = 1024; that is where the HODLR case runs."""
    from george_b200 import kernels as K
    rng = np.random.default_rng(9)
    x = np.sort(rng.uniform(0, 30, n))
    gp = _make_gp(solver_name, 1.0 * K.ExpSquaredKernel(1.0))
    gp.compute(x, 0.1)
    y = np.cos(x)
    t = rng.uniform(0, 30, 700)
    a = [gp.predict(y, t, return_var=True)[1], gp.predict(y, t)[1]]
    b = [gp.predict(y, t, return_var=True)[1], gp.predict(y, t)[1]]
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


@pytest.mark.parametrize("solver_name", ["basic", "hodlr"])
def test_edges_and_errors(gpu, env, solver_name):
    import george_b200 as george
    from george_b200 import kernels as K
    from george_b200._spec import DimensionMismatch
    kernel = 1.0 * K.ExpSquaredKernel(1.0)
    solver = george.BasicSolver if solver_name == "basic" else george.HODLRSolver
    with pytest.raises(RuntimeError):
        solver(kernel).predictive(kernel, np.zeros((3, 1)), "var")
    x = np.linspace(0, 5, 120)
    gp = george.GP(kernel, solver=solver)
    gp.compute(x, 0.1)
    y = np.sin(x)
    for t in (np.zeros(0), np.zeros((0, 1))):
        mu, var = gp.predict(y, t, return_var=True)
        _, cov = gp.predict(y, t)
        assert mu.shape == var.shape == (0,) and cov.shape == (0, 0)
    k3 = K.ExpSquaredKernel(1.0, ndim=3)
    with pytest.raises(DimensionMismatch):
        gp._predict_host(gp._compute_alpha(y, True), gp.parse_samples(x[:4]), True, k3)
    with pytest.raises(DimensionMismatch):
        gp.predict(y, x[:4], return_var=True, kernel=k3)
    with pytest.raises(ValueError):
        gp.solver.predictive(kernel, x[:4], "diag")


def test_pickled_dense_solver_takes_host_path(gpu, env):
    import george_b200 as george
    from george_b200 import kernels as K
    x = np.linspace(0, 5, 150)
    y = np.sin(x)
    gp = george.GP(0.5 * K.Matern32Kernel(0.3), solver=george.BasicSolver)
    gp.compute(x, 0.05)
    t = np.linspace(-0.5, 5.5, 40)
    _, var0 = gp.predict(y, t, return_var=True)
    _, cov0 = gp.predict(y, t)
    gp2 = pickle.loads(pickle.dumps(gp, -1))
    assert gp2.solver.predictive(gp2.kernel, t[:, None], "var") is None
    _, var1 = gp2.predict(y, t, return_var=True)
    _, cov1 = gp2.predict(y, t)
    kss = gp.kernel.get_value(t[:, None])
    assert _err(var1, var0, kss) <= HOST_TOL and _err(cov1, cov0, kss) <= HOST_TOL


def test_plugin_solver_without_predictive_takes_host_path(gpu, env):
    import george_b200 as george
    from george_b200 import kernels as K

    calls = []

    class Plugin(george.BasicSolver):
        predictive = None

        def apply_inverse(self, y, in_place=False):
            calls.append(np.shape(y))
            return super(Plugin, self).apply_inverse(y, in_place=in_place)

    x = np.linspace(0, 5, 100)
    y = np.sin(x)
    gp = george.GP(1.0 * K.ExpSquaredKernel(1.0), solver=Plugin)
    gp.compute(x, 0.1)
    t = np.linspace(0, 5, 13)
    _, var = gp.predict(y, t, return_var=True)
    assert (100, 13) in calls
    ref = george.GP(1.0 * K.ExpSquaredKernel(1.0))
    ref.compute(x, 0.1)
    _, var_d = ref.predict(y, t, return_var=True)
    assert _err(var, var_d, gp.kernel.get_value(t[:, None])) <= HOST_TOL


def test_abi_errors(gpu):
    import george_b200 as george
    from george_b200 import _lib, kernels as K
    from george_b200._spec import flatten
    lib = _lib.load()
    kernel = 1.0 * K.ExpSquaredKernel(1.0)
    spec = flatten(kernel)
    x = np.linspace(0, 5, 80)
    s = george.BasicSolver(kernel)
    s.compute(x[:, None], 0.1 * np.ones(80))
    xs = np.linspace(0, 5, 4)[:, None].copy()
    out = np.zeros(16)
    assert lib.bgp_dense_predict(s._handle.ptr, C.byref(spec), _lib.ptr(xs), 4, 2, _lib.ptr(out)) == _lib.BGP_ERR_INVALID
    assert lib.bgp_dense_predict(s._handle.ptr, C.byref(spec), _lib.ptr(xs), -1, 0, _lib.ptr(out)) == _lib.BGP_ERR_INVALID
    spec3 = flatten(K.ExpSquaredKernel(1.0, ndim=3))
    assert lib.bgp_dense_predict(s._handle.ptr, C.byref(spec3), _lib.ptr(xs), 4, 0, _lib.ptr(out)) == _lib.BGP_ERR_DIM
    assert lib.bgp_dense_predict(s._handle.ptr, C.byref(spec), _lib.ptr(xs), 0, 1, _lib.ptr(out)) == _lib.BGP_OK
    s2 = pickle.loads(pickle.dumps(s, -1))  # restored through bgp_dense_import_factor
    assert lib.bgp_dense_predict(s2._handle.ptr, C.byref(spec), _lib.ptr(xs), 4, 0, _lib.ptr(out)) == _lib.BGP_ERR_NOT_COMPUTED
    h = george.HODLRSolver(kernel, min_size=20)
    h.compute(x[:, None], 0.1 * np.ones(80))
    p = h.solver._ptr
    assert lib.bgp_hodlr_predict(p, C.byref(spec), _lib.ptr(xs), 4, 5, _lib.ptr(out)) == _lib.BGP_ERR_INVALID
    assert lib.bgp_hodlr_predict(p, C.byref(spec3), _lib.ptr(xs), 4, 1, _lib.ptr(out)) == _lib.BGP_ERR_DIM
    fresh = C.c_void_p()
    _lib.check(lib.bgp_hodlr_create(C.byref(fresh)))
    assert lib.bgp_hodlr_predict(fresh, C.byref(spec), _lib.ptr(xs), 4, 0, _lib.ptr(out)) == _lib.BGP_ERR_NOT_COMPUTED
    lib.bgp_hodlr_destroy(fresh)
