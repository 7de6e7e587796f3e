# -*- coding: utf-8 -*-
"""Leave-one-out cross-validation on the device: ``bgp_dense_loo_terms`` and ``bgp_hodlr_loo_terms`` (csrc/dense.cu,
csrc/hodlr.cu) and ``GP.loo_predict`` / ``GP.loo_log_likelihood`` / ``GP.grad_loo_log_likelihood`` on top of them.

* dense: the LOO predictive and value against a longdouble brute-force refit of N - 1 points (tests/hiprec.py), the
  gradient against the longdouble formula with the device's dK (``bgp_kmat_gradient_symmetric``) and against centred
  differences of the brute-force value, over 1-D ExpSquared, 3-D axis-aligned Matern52, a sum times a product and a
  generated user kernel;
* HODLR on exact-K trees (``ExpKernel`` on sorted 1-D inputs, ``exhaust="dense"``: the HODLR matrix is K) against the
  same longdouble references over slab widths 64, 192 (ragged tail) and the default; ``d`` against ``get_inverse()`` of
  the same handle, and two calls bit for bit;
* the GP layer: value == ``grad_loo_log_likelihood(return_value=True)[0]`` bit for bit, the host route of a pickled
  dense solver, a non-positive-definite K, a NaN mean, more than 64 kernel parameters and the error returns.
"""
import pickle

import numpy as np
import pytest

import hiprec

pytestmark = pytest.mark.gpu

LD = np.longdouble

# bars: 10-60x the largest value measured on one H100 80GB HBM3 (SXM, 700 W power limit)
DENSE_PRED_TOL = 2e-12    # mu, var vs the longdouble refit, relative to max |ref|           (measured 5.7e-14)
DENSE_VALUE_TOL = 1e-12   # value vs longdouble, relative                                      (measured 2.8e-14)
DENSE_GRAD_TOL = 2e-11    # g, diagA, beta vs the longdouble formula (g / sum |dK| |A|)        (measured 6.9e-13)
FD_TOL = 2e-8             # gradient vs centred differences of the brute-force value          (measured 7.9e-10)
HODLR_TOL = 1e-10         # alpha, d, beta, g, diagA vs longdouble on exact-K trees           (measured 2.7e-12)
HOST_ROUTE_TOL = 2e-13    # pickled dense solver (host route) vs the device route             (measured 8.5e-15)

BGP_OK, BGP_ERR_INVALID, BGP_ERR_NOT_COMPUTED = 0, 1, 3


@pytest.fixture
def env(monkeypatch):
    for var in ("BGP_GRAD_CHUNK", "BGP_SMALL_RANK_LIMIT", "BGP_PREDICT_CHUNK"):
        monkeypatch.delenv(var, raising=False)
    return monkeypatch


def _dense_kernels():
    from george_b200 import kernels as K
    return {
        "expsq_1d": (1.5 * K.ExpSquaredKernel(0.5), 1),
        "m52_3d_axis": (0.8 * K.Matern52Kernel([0.5, 1.0, 2.0], ndim=3), 3),
        "sum_x_prod": ((1.0 * K.ExpSquaredKernel(1.0, ndim=2) + 0.4 * K.Matern32Kernel(2.0, ndim=2))
                       * K.RationalQuadraticKernel(log_alpha=0.3, metric=1.5, ndim=2), 2),
        "user_cauchy": (0.8 * K.CauchyKernel(metric=0.7, ndim=2), 2),
    }


def _inputs(n, ndim, seed=0):
    rng = np.random.default_rng(seed + 7 * n + ndim)
    x = rng.uniform(0, 3, (n, ndim))
    yerr = 0.1 + 0.05 * rng.random(n)
    y = np.sin(2.0 * x[:, 0]) + 0.1 * rng.standard_normal(n)
    return x, yerr, y


def _kmat(kernel, x, yerr):
    K = kernel.get_value(x)
    K[np.diag_indices(len(x))] += yerr ** 2
    return K


def _ld_formula(K, r, dK=None):
    """The LOO terms of K in longdouble: alpha, d, beta, A, value, and g = einsum(dK, A) with its scale."""
    n = K.shape[0]
    Kinv = hiprec.solve_ld(hiprec.chol_ld(K), np.eye(n))
    Kinv = (Kinv + Kinv.T) / 2
    alpha = Kinv @ np.asarray(r, dtype=LD)
    d = np.diag(Kinv).copy()
    q = alpha / d
    beta = Kinv @ q
    c = (1 + alpha * q) / (2 * d)
    A = (np.outer(beta, alpha) + np.outer(alpha, beta)) / 2 - Kinv @ (c[:, None] * Kinv)
    value = np.sum(-np.log(2 * np.pi * np.ones(1, dtype=LD)) / 2 + np.log(d) / 2 - alpha ** 2 / (2 * d))
    out = dict(alpha=alpha, d=d, beta=beta, A=A, value=value)
    if dK is not None:
        dK = np.asarray(dK, dtype=LD)
        out["g"] = np.einsum("ijk,ij->k", dK, A)
        scale = np.einsum("ijk,ij->k", np.abs(dK), np.abs(A))
        scale[scale == 0] = 1
        out["gscale"] = scale
    return out


def _brute_ld(K, r, points):
    """The LOO predictive (mu - mean, var) at ``points`` by refitting N - 1 points in longdouble, and the value summed
    over ``points``."""
    n = K.shape[0]
    mu, var = [], []
    for i in points:
        k = np.delete(np.arange(n), i)
        if len(k) == 0:
            m, v = LD(0), LD(K[i, i])
        else:
            L = hiprec.chol_ld(K[np.ix_(k, k)])
            m = np.asarray(K[i, k], dtype=LD) @ hiprec.solve_ld(L, np.asarray(r[k], dtype=LD))
            v = LD(K[i, i]) - np.asarray(K[i, k], dtype=LD) @ hiprec.solve_ld(L, np.asarray(K[k, i], dtype=LD))
        mu.append(m)
        var.append(v)
    mu, var = np.array(mu, dtype=LD), np.array(var, dtype=LD)
    res = np.asarray(r, dtype=LD)[list(points)] - mu
    value = np.sum(-np.log(2 * np.pi * var) / 2 - res ** 2 / (2 * var))
    return mu, var, value


def _rel(a, ref):
    ref = np.asarray(ref, dtype=LD)
    den = np.max(np.abs(ref))
    return float(np.max(np.abs(np.asarray(a, dtype=LD) - ref)) / (den if den > 0 else 1))


def _points(n):
    return list(range(n)) if n <= 33 else sorted({0, 1, n // 3, n // 2, n - 2, n - 1})


# ---- 1. dense ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [1, 2, 33, 257])
@pytest.mark.parametrize("name", ["expsq_1d", "m52_3d_axis", "sum_x_prod", "user_cauchy"])
def test_dense_against_longdouble(gpu, record_property, name, n):
    from george_b200 import BasicSolver
    kernel, ndim = _dense_kernels()[name]
    x, yerr, y = _inputs(n, ndim)
    s = BasicSolver(kernel)
    s.compute(x, yerr)
    which = np.ones(len(kernel.get_parameter_vector(include_frozen=True)), dtype=np.uint32)
    alpha, d, beta, g, diag = s.loo_terms(y, which)
    a2, d2 = s.loo_terms(y)
    assert np.array_equal(a2, alpha) and np.array_equal(d2, d)
    K = _kmat(kernel, x, yerr)
    ref = _ld_formula(K, y, kernel.get_gradient(x, include_frozen=True))
    pts = _points(n)
    mu_b, var_b, val_b = _brute_ld(K, y, pts)
    mu = (y - alpha / d)[pts]
    var = (1.0 / d)[pts]
    errs = {
        "pred": max(_rel(mu, mu_b), _rel(var, var_b)),
        "value": abs(float(np.sum(-0.5 * np.log(2 * np.pi) + 0.5 * np.log(d) - alpha ** 2 / (2 * d)) - ref["value"]))
        / abs(float(ref["value"])),
        "grad": max(float(np.max(np.abs(g - ref["g"]) / ref["gscale"])), _rel(diag, np.diag(ref["A"])),
                    _rel(beta, ref["beta"])),
    }
    if n <= 33:  # the brute force covers every point: the formula's value is the refit's
        errs["value"] = max(errs["value"], float(abs(ref["value"] - val_b) / abs(val_b)))
    record_property("loo_err", errs)
    assert errs["pred"] <= DENSE_PRED_TOL and errs["value"] <= DENSE_VALUE_TOL and errs["grad"] <= DENSE_GRAD_TOL, errs


@pytest.mark.parametrize("name", ["expsq_1d", "user_cauchy"])
def test_dense_gradient_against_centred_differences(gpu, record_property, name):
    """The GP gradient (kernel, a fitted white noise and a fitted constant mean) against centred differences of the
    longdouble brute-force LOO value."""
    import george_b200 as george
    kernel, ndim = _dense_kernels()[name]
    x, yerr, y = _inputs(33, ndim, seed=1)
    gp = george.GP(kernel, mean=0.2, fit_mean=True, white_noise=np.log(0.02), fit_white_noise=True)
    gp.compute(x, yerr)
    v0 = gp.get_parameter_vector()
    value, grad = gp.grad_loo_log_likelihood(y, return_value=True)

    def brute(v):
        gp.set_parameter_vector(v)
        K = gp.get_matrix(x)
        K[np.diag_indices(len(x))] += yerr ** 2 + np.exp(gp.white_noise.get_value(x))
        return float(_brute_ld(K, y - gp.mean.get_value(x), range(len(x)))[2])

    assert abs(value - brute(v0)) <= DENSE_VALUE_TOL * abs(value)
    h = 1e-5
    fd = np.array([(brute(v0 + h * e) - brute(v0 - h * e)) / (2 * h) for e in np.eye(len(v0))])
    gp.set_parameter_vector(v0)
    err = float(np.max(np.abs(grad - fd) / np.maximum(1, np.abs(grad))))
    record_property("fd_err", err)
    assert err <= FD_TOL, (grad, fd)


# ---- 2. HODLR on exact-K trees ---------------------------------------------------------------------------------------

def _exp_case(n):
    from george_b200 import kernels as K
    kernel = 1.0 * K.ExpKernel(1.0)
    rng = np.random.default_rng(11 + n)
    x = np.sort(rng.uniform(0, n / 50.0, n))[:, None]
    yerr = 0.1 * np.ones(n)
    y = np.sin(3.0 * x[:, 0]) + 0.5
    return kernel, x, yerr, y


@pytest.mark.parametrize("chunk", ["64", "192", None])
@pytest.mark.parametrize("n,min_size", [(257, 32), (700, 50)])
def test_hodlr_exact_tree(gpu, env, record_property, n, min_size, chunk):
    import george_b200 as george
    kernel, x, yerr, y = _exp_case(n)
    if chunk is not None:
        env.setenv("BGP_GRAD_CHUNK", chunk)
    s = george.HODLRSolver(kernel, min_size=min_size, tol=1e-12, seed=42, rng_mode="pernode", exhaust="dense")
    s.compute(x, yerr)
    which = np.ones(2, dtype=np.uint32)
    alpha, d, beta, g, diag = s.loo_terms(y, which)
    again = s.loo_terms(y, which)
    for a, b in zip((alpha, d, beta, g, diag), again):  # n <= 1024: the solve has no atomics
        assert np.array_equal(a, b)
    a1, d1 = s.loo_terms(y)
    assert np.array_equal(a1, alpha) and np.array_equal(d1, d)
    assert np.array_equal(d, np.diag(s.get_inverse()))  # the restricted solve is the full one, bit for bit
    ref = _ld_formula(_kmat(kernel, x, yerr), y, kernel.get_gradient(x, include_frozen=True))
    errs = {"alpha": _rel(alpha, ref["alpha"]), "d": _rel(d, ref["d"]), "beta": _rel(beta, ref["beta"]),
            "g": float(np.max(np.abs(g - ref["g"]) / ref["gscale"])), "diag": _rel(diag, np.diag(ref["A"]))}
    record_property("loo_err", errs)
    assert max(errs.values()) <= HODLR_TOL, errs


def test_hodlr_slab_width_does_not_change_g(gpu, env):
    """The contraction's sum order depends only on n: g from 64- and 192-column slabs agrees to rounding of the solves
    (the T slabs are solved in different column groups) and diagA is the same entries."""
    import george_b200 as george
    kernel, x, yerr, y = _exp_case(700)
    s = george.HODLRSolver(kernel, min_size=50, tol=1e-12, seed=42, rng_mode="pernode", exhaust="dense")
    s.compute(x, yerr)
    out = {}
    for chunk in ("64", "192"):
        env.setenv("BGP_GRAD_CHUNK", chunk)
        out[chunk] = s.loo_terms(y, np.ones(2, dtype=np.uint32))
    assert np.array_equal(out["64"][1], out["192"][1])
    assert np.allclose(out["64"][3], out["192"][3], rtol=1e-12, atol=0)


# ---- 3. the GP layer -------------------------------------------------------------------------------------------------

def _gp(solver, n=300, **kw):
    import george_b200 as george
    from george_b200 import kernels as K
    rng = np.random.default_rng(5)
    x = np.sort(rng.uniform(0, 10, n))
    y = np.sin(x) + 0.1 * rng.standard_normal(n)
    gp = george.GP(0.8 * K.Matern32Kernel(1.5), mean=0.1, fit_mean=True, white_noise=np.log(0.01),
                   fit_white_noise=True, solver=solver, **kw)
    gp.compute(x, 0.05)
    return gp, y


def _solvers():
    import george_b200 as george
    return [(george.BasicSolver, {}), (george.HODLRSolver, dict(min_size=64, tol=1e-12))]


@pytest.mark.parametrize("which", [0, 1])
def test_value_is_return_value_bit_for_bit(gpu, which):
    solver, kw = _solvers()[which]
    gp, y = _gp(solver, **kw)
    value = gp.loo_log_likelihood(y)
    v2, grad = gp.grad_loo_log_likelihood(y, return_value=True)
    assert np.isfinite(value) and v2 == value
    assert np.array_equal(grad, gp.grad_loo_log_likelihood(y))
    mu, var = gp.loo_predict(y)
    assert mu.shape == var.shape == (len(y),) and np.all(var > 0)


def test_hodlr_agrees_with_dense(gpu):
    """At tol = 1e-12 the HODLR matrix is K to ~1e-12: its LOO terms are the dense ones to that accuracy."""
    import george_b200 as george
    gd, y = _gp(george.BasicSolver)
    gh, _ = _gp(george.HODLRSolver, min_size=64, tol=1e-12)
    vd, g_d = gd.grad_loo_log_likelihood(y, return_value=True)
    vh, g_h = gh.grad_loo_log_likelihood(y, return_value=True)
    assert abs(vd - vh) <= 1e-8 * abs(vd)
    assert np.allclose(g_d, g_h, rtol=1e-6, atol=1e-6 * np.max(np.abs(g_d)))
    for a, b in zip(gd.loo_predict(y), gh.loo_predict(y)):
        assert np.allclose(a, b, rtol=1e-8, atol=1e-10)


def test_pickled_dense_solver_takes_the_host_route(gpu, record_property):
    import george_b200 as george
    gp, y = _gp(george.BasicSolver)
    value, grad = gp.grad_loo_log_likelihood(y, return_value=True)
    mu, var = gp.loo_predict(y)
    gp2 = pickle.loads(pickle.dumps(gp, -1))
    gp2.recompute()
    assert gp2.solver.loo_terms(np.zeros(len(y))) is None  # no coordinates on the restored handle: host route
    v2, g2 = gp2.grad_loo_log_likelihood(y, return_value=True)
    mu2, var2 = gp2.loo_predict(y)
    errs = {"value": abs(v2 - value) / abs(value), "grad": float(np.max(np.abs(g2 - grad)) / np.max(np.abs(grad))),
            "pred": max(_rel(mu2, mu), _rel(var2, var))}
    record_property("host_route_err", errs)
    assert max(errs.values()) <= HOST_ROUTE_TOL, errs


@pytest.mark.parametrize("which", [0, 1])
def test_not_positive_definite(gpu, which):
    from numpy.linalg import LinAlgError
    import george_b200 as george
    from george_b200 import kernels as K
    solver, kw = _solvers()[which]
    x = np.linspace(0, 1, 50)
    gp = george.GP(K.DotProductKernel(), white_noise=0.0, fit_white_noise=True, solver=solver, **kw)
    gp.compute(x, 0.0)
    gp.set_parameter("white_noise:value", -80.0)  # rank-1 K without a noise floor: not positive definite
    y = np.sin(x)
    if which == 0:
        assert gp.loo_log_likelihood(y, quiet=True) == -np.inf
        assert np.array_equal(gp.grad_loo_log_likelihood(y, quiet=True), np.zeros(len(gp)))
        v, g = gp.grad_loo_log_likelihood(y, quiet=True, return_value=True)
        assert v == -np.inf and np.array_equal(g, np.zeros(len(gp)))
        with pytest.raises(LinAlgError):
            gp.loo_log_likelihood(y)
        with pytest.raises(LinAlgError):
            gp.grad_loo_log_likelihood(y)
    else:  # an LU-based HODLR matrix factorises; a d_i that is not positive is -inf / a ValueError naming the point
        try:
            gp.recompute(quiet=False)
        except (LinAlgError, ValueError):
            return
        v = gp.loo_log_likelihood(y, quiet=True)
        alpha, d = gp.solver.loo_terms(y - gp.mean.get_value(x))
        if np.all(np.isfinite(d) & (d > 0)):
            assert v == gp.loo_log_likelihood(y)
        else:
            assert v == -np.inf
            with pytest.raises(ValueError, match="point"):
                gp.grad_loo_log_likelihood(y)
            assert np.array_equal(gp.grad_loo_log_likelihood(y, quiet=True), np.zeros(len(gp)))


@pytest.mark.parametrize("which", [0, 1])
def test_nan_mean(gpu, which):
    solver, kw = _solvers()[which]
    gp, y = _gp(solver, **kw)
    gp.set_parameter("mean:value", np.nan)
    assert gp.loo_log_likelihood(y, quiet=True) == -np.inf
    assert np.array_equal(gp.grad_loo_log_likelihood(y, quiet=True), np.zeros(len(gp)))
    with pytest.raises(ValueError, match="mean function"):
        gp.loo_log_likelihood(y)
    with pytest.raises(ValueError, match="mean function"):
        gp.grad_loo_log_likelihood(y)


@pytest.mark.parametrize("which", [0, 1])
def test_more_than_64_kernel_parameters(gpu, which):
    """The gradient raises grad_log_likelihood's error; the value needs no contraction and runs."""
    import george_b200 as george
    from george_b200 import kernels as K
    solver, kw = _solvers()[which]
    kernel = K.Matern32Kernel([1.0] * 8, ndim=8)
    for _ in range(7):
        kernel = kernel + K.Matern32Kernel([1.0] * 8, ndim=8)
    kernel = kernel + K.ConstantKernel(log_constant=0.1, ndim=8)
    assert len(kernel) == 65
    rng = np.random.default_rng(0)
    x = rng.uniform(0, 1, (200, 8))
    y = np.sin(x[:, 0])
    gp = george.GP(kernel, solver=solver, **dict(kw, min_size=50) if kw else {})
    gp.compute(x, 0.1)
    with pytest.raises(ValueError, match="64") as exc_loo:
        gp.grad_loo_log_likelihood(y)
    with pytest.raises(ValueError, match="64") as exc_ll:
        gp.grad_log_likelihood(y)
    assert str(exc_loo.value) == str(exc_ll.value)
    assert np.isfinite(gp.loo_log_likelihood(y))


def _raw_loo(lib_fn, ptr, n, P, grad=True):
    from george_b200 import _lib
    which = np.ones(max(P, 1), dtype=np.uint32)
    r = np.ones(n)
    bufs = [np.zeros(n), np.zeros(n), np.zeros(n), np.zeros(max(P, 1)), np.zeros(n)]
    ptrs = [_lib.ptr(b) for b in bufs]
    if not grad:
        ptrs[2:] = [None, None, None]
    st = lib_fn(ptr, _lib.ptr(which), _lib.ptr(r), *ptrs)
    return st, _lib.last_error()


def test_errors(gpu):
    from george_b200 import _lib
    from george_b200.solvers._hodlr import HODLRSolver as Native
    import test_gpu_hodlr_shards as sh
    lib = _lib.load()
    import ctypes as C
    ptr = C.c_void_p()
    _lib.check(lib.bgp_dense_create(C.byref(ptr)))
    try:
        assert _raw_loo(lib.bgp_dense_loo_terms, ptr, 8, 2) == (BGP_ERR_NOT_COMPUTED, "the solver has not been computed")
    finally:
        lib.bgp_dense_destroy(ptr)
    Native.release_parked()
    fresh = Native()
    assert _raw_loo(lib.bgp_hodlr_loo_terms, fresh._ptr, 8, 2) == (BGP_ERR_NOT_COMPUTED,
                                                                   "the solver has not been computed")
    kernel, x, yerr, _ = _exp_case(1024)
    shards = sh._shards(kernel, x, yerr, 2, min_size=32, tol=1e-12)
    for s in shards.handles:
        assert _raw_loo(lib.bgp_hodlr_loo_terms, s._ptr, 1024, 2) == (
            BGP_ERR_INVALID, "loo_terms is not available on a sharded factorisation")


def test_exported_dense_factor_is_not_computed_for_loo(gpu):
    """A dense handle loaded by bgp_dense_import_factor holds no kernel or coordinates, as bgp_dense_grad_terms says."""
    import ctypes as C
    import george_b200 as george
    from george_b200 import _lib
    gp, y = _gp(george.BasicSolver, n=64)
    lib = _lib.load()
    n = len(y)
    factor = np.zeros(n * n)
    _lib.check(lib.bgp_dense_export_factor(gp.solver._handle.ptr, _lib.ptr(factor)))
    ptr = C.c_void_p()
    _lib.check(lib.bgp_dense_create(C.byref(ptr)))
    try:
        _lib.check(lib.bgp_dense_import_factor(ptr, _lib.ptr(factor), n, C.c_double(0.0)))
        st, msg = _raw_loo(lib.bgp_dense_loo_terms, ptr, n, 3, grad=False)
        assert st == BGP_ERR_NOT_COMPUTED and "imported" in msg
    finally:
        lib.bgp_dense_destroy(ptr)
