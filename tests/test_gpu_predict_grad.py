# -*- coding: utf-8 -*-
"""GP.grad_predict on the device: gradients of the predictive mean and variance with respect to the test points
(``bgp_kmat_x1_gradient_matvec``, ``bgp_dense_predict_grad``, ``bgp_hodlr_predict_grad``; csrc/kmat_ops.cu, dense.cu,
hodlr.cu).

Finite-difference tolerance.  Every check moves all test points along one axis by +-h and takes
``(f(t + h) - f(t - h)) / 2h``.  Its truncation error is ``h^2 |f'''| / 6``; with h = 1e-5 and length scales >= 0.3
that is below 1e-8 of the prior scale.  Its rounding error is ``delta / h``, delta being the error of one ``predict``:
about 1e-15 of the prior scale for mu and var (1e-13 is the bar of tests/test_gpu_predict.py), so below 1e-8 as well.
The bar FD_TOL = 1e-7 of the scale ``max(1, |k**|, |f'|)`` is 30x the largest error measured on one H100 80GB HBM3
(SXM, 700 W power limit), 3.2e-9; the general-metric error this feature fixes is 0.54 on that scale.
"""
import pickle

import numpy as np
import pytest

import hiprec

pytestmark = pytest.mark.gpu

LD = np.longdouble
FD_H = 1e-5
FD_TOL = 1e-7
# At N = 2^18 the mean sums 2^18 terms with |alpha| up to ~1e2: predict's rounding is ~1e-11 and h = 1e-4 (length
# scale 2) makes the difference quotient's rounding ~1e-7 (measured 1.6e-7)
HEADLINE_FD_TOL = 2e-6
# dense vs the longdouble reference.  alpha and W = K^-1 K(x, x*) carry up to cond(K) * eps of forward error; at
# n = 300, yerr = 0.3 and a unit prior cond(K) <= 1 + 300 / 0.09 ~ 3.4e3, i.e. ~8e-13; measured 2.5e-15.  Relative to
# max |reference|:
HIPREC_TOL = 1e-13
ROUTE_TOL = 1e-13       # host route vs device route on the same factorisation            (measured 3.6e-15)
HODLR_EXACT_TOL = 1e-8  # HODLR at tol = 1e-12 vs dense                                    (measured 6.7e-10)


@pytest.fixture
def env(monkeypatch):
    for var in ("BGP_PREDICT_CHUNK", "BGP_DENSE_OB"):
        monkeypatch.delenv(var, raising=False)
    return monkeypatch


def _points(ndim, n, rng, lo=-1.5, hi=1.5):
    x = rng.uniform(lo, hi, (n, ndim))
    return x[np.argsort(x[:, 0])]


def _arg(x):
    return x[:, 0] if x.shape[1] == 1 else x


def _zoo():
    from conftest import make_kernels
    from george_b200 import kernels as K
    zoo = list(make_kernels())
    zoo.append(("cauchy_2d", 0.7 * K.CauchyKernel(1.3, ndim=2)
                + K.DampedCosineKernel(log_period=0.1, log_decay=0.7, ndim=2, axes=[0, 1])))
    zoo.append(("damped_cos_1d", 1.0 * K.CauchyKernel(metric=1.0)
                + 0.5 * K.DampedCosineKernel(log_period=np.log(3.0), log_decay=np.log(20.0))))
    return zoo


def _gp(kernel, solver="basic", **kw):
    import george_b200 as george
    s = {"basic": george.BasicSolver, "hodlr": george.HODLRSolver}[solver]
    return george.GP(kernel, solver=s, **kw)


def _fd(gp, y, t, h=FD_H, kernel=None):
    """Central differences of the device predict: (dmu, dvar), each (ns, ndim)."""
    t = np.asarray(t, dtype=np.float64).reshape(len(t), -1)
    dmu, dvar = np.empty(t.shape), np.empty(t.shape)
    for q in range(t.shape[1]):
        tp, tm = t.copy(), t.copy()
        tp[:, q] += h
        tm[:, q] -= h
        mp, vp = gp.predict(y, _arg(tp), return_var=True, kernel=kernel)
        mm, vm = gp.predict(y, _arg(tm), return_var=True, kernel=kernel)
        dmu[:, q] = 0.5 * (mp - mm) / h
        dvar[:, q] = 0.5 * (vp - vm) / h
    return dmu, dvar


def _fd_err(gp, y, t, kernel=None):
    k = gp.kernel if kernel is None else kernel
    mu, var, dmu, dvar = gp.grad_predict(y, t, return_var=True, kernel=kernel)
    fmu, fvar = _fd(gp, y, np.asarray(t).reshape(len(t), -1), kernel=kernel)
    t2 = np.asarray(t, dtype=np.float64).reshape(len(t), -1)
    scale = max(1.0, float(np.max(np.abs(k.get_value(t2, diag=True)))), float(np.max(np.abs(fmu))),
                float(np.max(np.abs(fvar))))
    return max(float(np.max(np.abs(dmu - fmu))), float(np.max(np.abs(dvar - fvar)))) / scale


# ---- 1. bit parity with predict ----------------------------------------------------------------------------------
@pytest.mark.parametrize("solver", ["basic", "hodlr"])
@pytest.mark.parametrize("idx", range(16))
def test_mu_and_var_bit_for_bit_predict(gpu, env, idx, solver):
    name, kernel = _zoo()[idx]
    rng = np.random.default_rng(500 + idx)
    x = _points(kernel.ndim, 300, rng)
    y = np.sin(3 * x[:, 0])
    t = _arg(_points(kernel.ndim, 70, rng))
    gp = _gp(kernel, solver, **({"min_size": 40} if solver == "hodlr" else {}))
    gp.compute(_arg(x), 0.3)
    mu, var, dmu, dvar = gp.grad_predict(y, t, return_var=True)
    mu2, dmu2 = gp.grad_predict(y, t)
    assert np.array_equal(mu, gp.predict(y, t, return_cov=False)) and np.array_equal(mu, mu2)
    assert np.array_equal(var, gp.predict(y, t, return_var=True)[1])
    assert dmu.shape == dvar.shape == (len(t), kernel.ndim) and var.shape == mu.shape == (len(t),)
    assert np.all(np.isfinite(dmu)) and np.all(np.isfinite(dvar))
    if solver == "basic":  # identical calls, identical bits (the HODLR solve adds with atomics past 512 rows)
        again = gp.grad_predict(y, t, return_var=True)
        assert np.array_equal(again[2], dmu) and np.array_equal(again[3], dvar) and np.array_equal(dmu2, dmu)


@pytest.mark.parametrize("solver", ["basic", "hodlr"])
def test_kernel_override(gpu, env, solver):
    from george_b200 import kernels as K
    rng = np.random.default_rng(7)
    x = np.sort(rng.uniform(0, 10, 400))
    y = np.sin(x) + 0.1 * rng.normal(size=x.size)
    k1 = 1.5 * K.Matern32Kernel(2.0)
    k2 = 0.4 * K.ExpSine2Kernel(gamma=2.0, log_period=np.log(3.0))
    gp = _gp(k1 + k2, solver, mean=0.2, white_noise=np.log(0.05), **({"min_size": 40} if solver == "hodlr" else {}))
    gp.compute(x, 0.1)
    t = np.linspace(-1, 11, 90)
    for kern in (k1, k2):
        mu, var, dmu, dvar = gp.grad_predict(y, t, return_var=True, kernel=kern)
        assert np.array_equal(mu, gp.predict(y, t, return_cov=False, kernel=kern))
        assert np.array_equal(var, gp.predict(y, t, return_var=True, kernel=kern)[1])
        if solver == "basic":
            assert _fd_err(gp, y, t, kernel=kern) <= FD_TOL
    # the components' mean gradients add up to the full one (the mean is linear in the kernel)
    d1 = gp.grad_predict(y, t, kernel=k1)[1]
    d2 = gp.grad_predict(y, t, kernel=k2)[1]
    d = gp.grad_predict(y, t)[1]
    assert np.max(np.abs(d1 + d2 - d)) <= 1e-12 * max(1.0, np.max(np.abs(d)))


# ---- 2. finite differences ---------------------------------------------------------------------------------------
def _fd_cases():
    from george_b200 import kernels as K
    return [
        ("expsq_1d", 1.3 * K.ExpSquaredKernel(0.8), 1),
        ("m32_1d", 2.3 * K.Matern32Kernel(0.7), 1),
        ("m52_1d", K.Matern52Kernel(0.5), 1),
        ("exp_1d", 0.9 * K.ExpKernel(1.2), 1),
        ("ratquad_1d", K.RationalQuadraticKernel(log_alpha=0.3, metric=1.2), 1),
        ("expsq_3d_iso", K.ExpSquaredKernel(0.9, ndim=3), 3),
        ("m52_3d_axis", K.Matern52Kernel([0.5, 1.0, 2.0], ndim=3), 3),
        ("expsq_3d_general", K.ExpSquaredKernel([[1.0, 0.1, 0.2], [0.1, 2.0, 0.3], [0.2, 0.3, 1.5]], ndim=3), 3),
        ("m32_2d_general", K.Matern32Kernel([[2.0, 0.7], [0.7, 1.5]], ndim=2), 2),
        ("linear_1d", K.LinearKernel(log_gamma2=0.2, order=2), 1),
        ("poly_3d", K.PolynomialKernel(log_sigma2=0.1, order=3, ndim=3), 3),
        ("dot_2d", K.DotProductKernel(ndim=2) + K.ExpSquaredKernel(1.0, ndim=2), 2),
        ("localgauss_1d", K.LocalGaussianKernel(location=0.1, log_width=0.2) + 0.5 * K.Matern52Kernel(1.0), 1),
        ("cosine_expsine2_1d", 0.5 * K.CosineKernel(log_period=0.5)
         + K.ExpSine2Kernel(gamma=1.0, log_period=np.log(3.0)), 1),
        ("expsq_block_3d", K.ExpSquaredKernel(1.0, ndim=3, block=[(-0.5, 0.5)] * 3), 3),
        ("sum_expsq_expsine2", 1.0 * K.ExpSquaredKernel(1.0, ndim=3)
         + 0.5 * K.ExpSine2Kernel(gamma=1.0, log_period=np.log(3.0), ndim=3, axes=1), 3),
        ("quasiperiodic_1d", 1.0 * K.ExpSquaredKernel(1.0) * K.ExpSine2Kernel(gamma=1.0, log_period=np.log(3.0)), 1),
        ("cos_x_localgauss", K.CosineKernel(log_period=0.5, ndim=3, axes=0)
         * K.LocalGaussianKernel(location=0.1, log_width=0.2, ndim=3, axes=1) + K.Matern32Kernel(1.0, ndim=3), 3),
        ("poly_lin_dot", K.PolynomialKernel(log_sigma2=0.1, order=3, ndim=3)
         + K.LinearKernel(log_gamma2=0.2, order=2, ndim=3) + K.DotProductKernel(ndim=3), 3),
        ("const_plus", 0.3 + K.Matern32Kernel(2.0, ndim=2), 2),
        ("cauchy_2d", 0.7 * K.CauchyKernel(1.3, ndim=2)
         + K.DampedCosineKernel(log_period=0.1, log_decay=0.7, ndim=2, axes=[0, 1]), 2),
        ("damped_cos_1d", 1.0 * K.CauchyKernel(metric=1.0)
         + 0.5 * K.DampedCosineKernel(log_period=np.log(3.0), log_decay=np.log(20.0)), 1),
    ]


def _away_from_edges(x, edges=(-0.5, 0.5), gap=0.05):
    far = np.all(np.min(np.abs(x[:, :, None] - np.array(edges)[None, None, :]), axis=2) > gap, axis=1)
    return x[far]


@pytest.mark.parametrize("idx", range(22))
def test_finite_differences_dense(gpu, env, record_property, idx):
    name, kernel, nd = _fd_cases()[idx]
    rng = np.random.default_rng(900 + idx)
    x = _points(nd, 200, rng)
    t = _points(nd, 40, rng)
    if "block" in name:  # test points inside the block, training points on both sides, none near an edge
        x, t = _away_from_edges(_points(nd, 400, rng, -0.9, 0.9)), _points(nd, 40, rng, -0.45, 0.45)
    y = np.sin(2 * x[:, 0]) + 0.1 * rng.normal(size=len(x))
    gp = _gp(kernel, mean=0.4)
    gp.compute(_arg(x), 0.3)
    err = _fd_err(gp, y, _arg(t))
    record_property("fd_err", err)
    assert err <= FD_TOL, (name, err)


def test_general_metric_regression(gpu, env, oracle, record_property):
    """For a general metric the new gradient is the derivative; get_x1_gradient stays the reference's value (checked
    against the CPU oracle), so contracting it with alpha misses the derivative by O(1)."""
    from george_b200 import kernels as K
    from george_b200._spec import flatten
    kernel = K.ExpSquaredKernel(metric=[[2.0, 0.7], [0.7, 1.5]], ndim=2)
    rng = np.random.default_rng(3)
    x = _points(2, 150, rng)
    t = _points(2, 30, rng)
    y = np.sin(2 * x[:, 0]) + np.cos(x[:, 1])
    gp = _gp(kernel)
    gp.compute(x, 0.2)
    _, dmu = gp.grad_predict(y, t)
    fmu, _ = _fd(gp, y, t)
    scale = max(1.0, np.max(np.abs(fmu)))
    assert np.max(np.abs(dmu - fmu)) <= FD_TOL * scale
    g_ref = kernel.get_x1_gradient(t, x)
    assert np.allclose(g_ref, oracle.x_gradient_general(flatten(kernel), 1, t, x), rtol=1e-12, atol=1e-14)
    alpha = gp._compute_alpha(y, True)
    old = np.einsum("ijq,j->iq", g_ref, alpha)
    miss = float(np.max(np.abs(old - fmu)) / scale)
    record_property("x1_gradient_miss", miss)
    assert miss > 1e-2


def test_exp_kernel_at_a_training_point(gpu, env):
    from george_b200 import kernels as K
    rng = np.random.default_rng(4)
    x = np.sort(rng.uniform(0, 5, 100))
    y = np.sin(x)
    for solver in ("basic", "hodlr"):
        gp = _gp(0.9 * K.ExpKernel(1.2), solver, **({"min_size": 20} if solver == "hodlr" else {}))
        gp.compute(x, 0.1)
        t = np.concatenate([x[[3, 50, 99]], [2.5]])
        mu, var, dmu, dvar = gp.grad_predict(y, t, return_var=True)
        assert np.all(np.isfinite(dmu)) and np.all(np.isfinite(dvar)) and np.all(np.isfinite(var))
        # interpreter route (a program the shaped evaluator does not take) as well
        gp2 = _gp(K.ExpKernel(1.2) + K.ConstantKernel(log_constant=-2.0), solver,
                  **({"min_size": 20} if solver == "hodlr" else {}))
        gp2.compute(x, 0.1)
        out = gp2.grad_predict(y, t, return_var=True)
        assert all(np.all(np.isfinite(o)) for o in out)


# ---- 3. extended precision ---------------------------------------------------------------------------------------
def _hiprec_case(name):
    from george_b200 import kernels as K
    if name == "expsq_iso":
        return 1.2 * K.ExpSquaredKernel(0.7, ndim=2), 1.2, np.diag([0.7, 0.7]), "expsq"
    if name == "expsq_axis":
        return 1.2 * K.ExpSquaredKernel([0.7, 1.6], ndim=2), 1.2, np.diag([0.7, 1.6]), "expsq"
    if name == "expsq_general":
        M = np.array([[2.0, 0.7], [0.7, 1.5]])
        return 1.2 * K.ExpSquaredKernel(M, ndim=2), 1.2, M, "expsq"
    return 0.8 * K.Matern32Kernel(0.9), 0.8, np.array([[0.9]]), "m32"


@pytest.mark.parametrize("name", ["expsq_iso", "expsq_axis", "expsq_general", "m32_1d"])
def test_against_extended_precision(gpu, env, record_property, name):
    kernel, c, M, prof = _hiprec_case(name)
    nd = M.shape[0]
    rng = np.random.default_rng(77)
    n = 300
    x = _points(nd, n, rng, -3, 3)
    t = _points(nd, 50, rng, -3.5, 3.5)
    y = np.sin(2 * x[:, 0]) + 0.1 * rng.normal(size=n)
    gp = _gp(kernel)
    gp.compute(_arg(x), 0.3)
    mu, var, dmu, dvar = gp.grad_predict(y, _arg(t), return_var=True)

    K = kernel.get_value(x)
    K[np.diag_indices(n)] += gp._sigma(gp._x) ** 2
    L = hiprec.chol_ld(K)
    alpha = hiprec.solve_ld(L, y.astype(LD)).ravel()
    Kxs = kernel.get_value(t, x)
    W = hiprec.solve_ld(L, Kxs.T)                      # (n, ns)
    Minv = np.linalg.inv(M).astype(LD)
    d = t[:, None, :].astype(LD) - x[None, :, :].astype(LD)   # (ns, n, nd)
    Md = np.einsum("pq,ijq->ijp", Minv, d)
    r2 = np.einsum("ijq,ijq->ij", d, Md)
    if prof == "expsq":
        f1 = -0.5 * c * np.exp(-0.5 * r2)
    else:
        f1 = -1.5 * c * np.exp(-np.sqrt(3 * r2))
    g = 2 * f1[:, :, None] * Md                       # d k(t_i, x_j) / d t_i
    dmu_ref = np.einsum("ijq,j->iq", g, alpha)
    dvar_ref = -2 * np.einsum("ijq,ji->iq", g, W)
    e_mu = float(np.max(np.abs(dmu - dmu_ref)) / np.max(np.abs(dmu_ref)))
    e_var = float(np.max(np.abs(dvar - dvar_ref)) / np.max(np.abs(dvar_ref)))
    record_property("err_dmu", e_mu)
    record_property("err_dvar", e_var)
    assert e_mu <= HIPREC_TOL and e_var <= HIPREC_TOL, (e_mu, e_var)


# ---- 4. routes agree ---------------------------------------------------------------------------------------------
def _route_err(a, b):
    return float(np.max(np.abs(a - b)) / max(1.0, np.max(np.abs(b))))


def test_pickled_dense_solver_takes_host_route(gpu, env, record_property):
    from george_b200 import kernels as K
    rng = np.random.default_rng(12)
    x = _points(3, 250, rng)
    y = np.sin(3 * x[:, 0])
    t = _points(3, 33, rng)
    gp = _gp(K.Matern52Kernel([0.5, 1.0, 2.0], ndim=3) + K.LinearKernel(log_gamma2=0.2, order=2, ndim=3))
    gp.compute(x, 0.3)
    dev = gp.grad_predict(y, t, return_var=True)
    gp2 = pickle.loads(pickle.dumps(gp))
    assert gp2.solver.predictive_grad(gp2.kernel, t) is None
    host = gp2.grad_predict(y, t, return_var=True)
    errs = [_route_err(a, b) for a, b in zip(host, dev)]
    record_property("max_err", max(errs))
    assert max(errs) <= ROUTE_TOL, errs


def test_trivial_solver_has_zero_mean_gradient(gpu, env):
    import george_b200 as george
    gp = george.GP(mean=0.3, white_noise=np.log(0.2))
    rng = np.random.default_rng(2)
    x = np.sort(rng.uniform(0, 5, 40))
    gp.compute(x, 0.05)
    y = np.sin(x)
    t = np.linspace(0, 5, 6)
    mu, dmu = gp.grad_predict(y, t)
    assert np.array_equal(mu, gp.predict(y, t, return_cov=False))
    assert dmu.shape == (6, 1) and np.all(dmu == 0.0)


def test_hodlr_exact_matches_dense(gpu, env, record_property):
    from george_b200 import kernels as K
    rng = np.random.default_rng(21)
    x = np.sort(rng.uniform(0, 20, 1500))
    y = np.sin(x) + 0.1 * rng.normal(size=x.size)
    t = rng.uniform(-1, 21, 200)
    kernel = 1.0 * K.Matern32Kernel(2.0) + 0.3 * K.ExpSine2Kernel(gamma=1.0, log_period=np.log(4.0))
    gd = _gp(kernel)
    gd.compute(x, 0.2)
    gh = _gp(kernel, "hodlr", tol=1e-12, min_size=64)
    gh.compute(x, 0.2)
    a, b = gd.grad_predict(y, t, return_var=True), gh.grad_predict(y, t, return_var=True)
    errs = [_route_err(u, v) for u, v in zip(b, a)]
    record_property("max_err", max(errs))
    assert max(errs) <= HODLR_EXACT_TOL, errs


def test_hodlr_default_tol_matches_its_own_predict(gpu, env, record_property):
    """At the default tol the HODLR factorisation is another covariance; dmu and dvar are derivatives of what HODLR's
    own predict returns.  K_h^-1 is symmetric only to the ACA's accuracy, and dvar = -2 dB^T K_h^-1 B assumes the
    symmetric part, so dvar carries that asymmetry: its bar is the spread between K_h^-1 B and K_h^-T B."""
    from george_b200 import kernels as K
    rng = np.random.default_rng(22)
    x = np.sort(rng.uniform(0, 20, 1000))
    y = np.sin(x) + 0.1 * rng.normal(size=x.size)
    t = rng.uniform(0, 20, 40)
    gp = _gp(1.0 * K.Matern32Kernel(2.0), "hodlr", min_size=64)
    gp.compute(x, 0.2)
    mu, var, dmu, dvar = gp.grad_predict(y, t, return_var=True)
    fmu, fvar = _fd(gp, y, t)
    e_mu = float(np.max(np.abs(dmu - fmu)) / max(1.0, np.max(np.abs(fmu))))
    Kinv = gp.solver.get_inverse()
    asym = float(np.max(np.abs(Kinv - Kinv.T)) / np.max(np.abs(Kinv)))
    e_var = float(np.max(np.abs(dvar - fvar)) / max(1.0, np.max(np.abs(fvar))))
    record_property("err_dmu", e_mu)
    record_property("err_dvar", e_var)
    record_property("kinv_asymmetry", asym)
    assert e_mu <= FD_TOL, e_mu
    assert e_var <= FD_TOL + 10 * asym, (e_var, asym)


# ---- 5. scale -----------------------------------------------------------------------------------------------------
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


def test_headline_hodlr_4096(gpu, env, record_property):
    gp, x, y, rng = _headline_gp()
    t = rng.uniform(-5, 2005, 4096)
    mu, var, dmu, dvar = gp.grad_predict(y, t, return_var=True)
    assert dmu.shape == dvar.shape == (4096, 1)
    assert all(np.all(np.isfinite(o)) for o in (mu, var, dmu, dvar))
    pick = np.sort(rng.choice(4096, 8, replace=False))
    fmu, fvar = _fd(gp, y, t[pick], h=1e-4)
    e = max(float(np.max(np.abs(dmu[pick] - fmu))), float(np.max(np.abs(dvar[pick] - fvar))))
    record_property("fd_err", e)
    assert e <= HEADLINE_FD_TOL, e
    env.setenv("BGP_PREDICT_CHUNK", "640")  # chunks of 640 test points with a ragged tail, vs 512 by default
    forced = gp.grad_predict(y, t, return_var=True)
    errs = [_route_err(a, b) for a, b in zip(forced, (mu, var, dmu, dvar))]
    record_property("chunk_err", max(errs))
    assert max(errs) <= 1e-12, errs


@pytest.mark.parametrize("chunk", ["7", "64"])
def test_dense_forced_chunks(gpu, env, chunk):
    from george_b200 import kernels as K
    rng = np.random.default_rng(31)
    x = _points(3, 700, rng)
    y = np.sin(3 * x[:, 0])
    t = _points(3, 150, rng)
    gp = _gp(K.Matern52Kernel([0.5, 1.0, 2.0], ndim=3))
    gp.compute(x, 0.3)
    ref = gp.grad_predict(y, t, return_var=True)
    env.setenv("BGP_PREDICT_CHUNK", chunk)
    got = gp.grad_predict(y, t, return_var=True)
    assert np.array_equal(got[0], ref[0])
    assert max(_route_err(a, b) for a, b in zip(got, ref)) <= 1e-12


# ---- 6. edge cases -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("solver", ["basic", "hodlr"])
def test_edges_and_errors(gpu, env, solver):
    from george_b200 import kernels as K
    from george_b200.modeling import Model
    rng = np.random.default_rng(5)
    x = np.sort(rng.uniform(0, 5, 200))
    y = np.sin(x)
    gp = _gp(1.0 * K.ExpSquaredKernel(1.0), solver, **({"min_size": 40} if solver == "hodlr" else {}))
    gp.compute(x, 0.1)
    mu, var, dmu, dvar = gp.grad_predict(y, np.zeros(0), return_var=True)
    assert mu.shape == var.shape == (0,) and dmu.shape == dvar.shape == (0, 1)
    mu, dmu = gp.grad_predict(y, np.array([1.0]))
    assert mu.shape == (1,) and dmu.shape == (1, 1)
    with pytest.raises(ValueError, match="Dimension mismatch"):
        gp.grad_predict(y, np.zeros((3, 2)))
    with pytest.raises(ValueError, match="Dimension mismatch"):
        gp.grad_predict(np.zeros(7), np.zeros(3))

    class Line(Model):
        parameter_names = ("m", "b")

        def get_value(self, x):
            return self.m * x + self.b

    gl = _gp(1.0 * K.ExpSquaredKernel(1.0), solver, mean=Line(m=1.0, b=0.0),
             **({"min_size": 40} if solver == "hodlr" else {}))
    gl.compute(x, 0.1)
    with pytest.raises(NotImplementedError):
        gl.grad_predict(y, x[:3], return_var=True)
    g9 = _gp(K.ExpSquaredKernel(1.0, ndim=9, axes=[0, 4, 8]), solver, **({"min_size": 40} if solver == "hodlr" else {}))
    g9.compute(rng.uniform(size=(60, 9)), 0.1)
    with pytest.raises(ValueError, match="at most 8"):
        g9.grad_predict(np.zeros(60), rng.uniform(size=(3, 9)))
    with pytest.raises(ValueError, match="at most 8"):
        g9.solver.predictive_grad(g9.kernel, rng.uniform(size=(3, 9)))
    import george_b200 as george
    with pytest.raises(RuntimeError):
        george.GP(1.0 * K.ExpSquaredKernel(1.0)).grad_predict(y, x[:3])


def test_abi_errors(gpu):
    import ctypes as C
    from george_b200 import _lib, kernels as K
    from george_b200._spec import flatten
    lib = _lib.load()
    spec = flatten(K.ExpSquaredKernel(1.0, ndim=2))
    x1, x2, v = np.zeros((3, 2)), np.zeros((5, 2)), np.zeros(20)
    out = np.zeros(6)
    assert lib.bgp_kmat_x1_gradient_matvec(C.byref(spec), _lib.ptr(x1), 3, _lib.ptr(x2), 5, _lib.ptr(v), 4, 1.0, 0,
                                           _lib.ptr(out)) == _lib.BGP_ERR_DIM
    assert lib.bgp_kmat_x1_gradient_matvec(C.byref(spec), _lib.ptr(x1), -1, _lib.ptr(x2), 5, _lib.ptr(v), 0, 1.0, 0,
                                           _lib.ptr(out)) == _lib.BGP_ERR_INVALID
    # n2 == 0: the prior term alone (DotProduct: d (x . x) / dx = 2 x)
    sd = flatten(K.DotProductKernel(ndim=2))
    x1 = np.array([[1.0, 2.0], [3.0, -1.0], [0.5, 0.25]])
    assert lib.bgp_kmat_x1_gradient_matvec(C.byref(sd), _lib.ptr(x1), 3, _lib.ptr(x2), 0, _lib.ptr(v), 0, -2.0, 1,
                                           _lib.ptr(out)) == _lib.BGP_OK
    assert np.array_equal(out.reshape(3, 2), 2 * x1)
    h = C.c_void_p()
    assert lib.bgp_dense_create(C.byref(h)) == 0
    var, dvar = np.zeros(3), np.zeros(6)
    assert lib.bgp_dense_predict_grad(h, C.byref(spec), _lib.ptr(x1), 3, _lib.ptr(var),
                                      _lib.ptr(dvar)) == _lib.BGP_ERR_NOT_COMPUTED
    lib.bgp_dense_destroy(h)
