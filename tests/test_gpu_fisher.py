# -*- coding: utf-8 -*-
"""``GP.fisher_information``, the expected Fisher information of the hyper-parameters, on the device
(``bgp_dense_fisher_terms``):

1. dense ``F`` against a longdouble brute force of ``F_pq = dmu_p^T K^-1 dmu_q + 1/2 tr(K^-1 dK_p K^-1 dK_q)`` with
   ``dK`` from ``kernel.get_gradient``, over several kernels and every block type (a fitted non-constant mean, a fitted
   non-constant white noise, a frozen kernel parameter);
2. a derivative-free check: ``F`` is the Hessian of ``KL(N(mu0, K0) || N(mu(theta), K(theta)))`` at ``theta0``, and
   central second differences of that KL, computed in float64 from covariance values alone, match it;
3. the scale identity: with ``yerr = 0``, a kernel ``c * K0`` and a fitted constant white noise, ``dK_c + dK_w = K``, so
   the sum of ``F``'s (log c, white noise) block is N/2, at sizes whose products take the direct and split-K paths;
4. exact symmetry, positive semi-definiteness and bit-identical repeated calls;
5. ``grad`` from ``fisher_information(y)`` is ``grad_log_likelihood(y)``'s bits;
6. the host route (a plug-in without the hook, a pickled dense solver) against the device route;
7. ``HODLRSolver`` raising ``NotImplementedError``, and more than 64 kernel parameters raising ``ValueError``.
"""
import pickle

import numpy as np
import pytest
import scipy.linalg as sla

from hiprec import LD, chol_ld, solve_ld

pytestmark = pytest.mark.gpu

BRUTE_TOL = 1e-10   # F vs longdouble, relative to max |F|
KL_TOL = 1e-5       # F vs central second differences of the KL, relative to max |F|
SCALE_TOL = 1e-11   # sum of the (log c, white noise) block vs N / 2, relative
HOST_TOL = 1e-11    # host route vs device route, relative to max |F|
PSD_TOL = 1e-12     # min eigenvalue >= -PSD_TOL * ||F||


def _line_mean(m, b):
    from george_b200.modeling import Model

    class LineMean(Model):
        parameter_names = ("m", "b")

        def get_value(self, x):
            return self.m * np.asarray(x).flatten() + self.b

        def compute_gradient(self, x):
            x = np.asarray(x).flatten()
            return np.vstack([x, np.ones_like(x)])

    return LineMean(m=m, b=b)


def _log_linear_noise(a, s):
    from george_b200.modeling import Model

    class LogLinearNoise(Model):
        parameter_names = ("a", "s")

        def get_value(self, x):
            return self.a + self.s * np.asarray(x).flatten()

        def compute_gradient(self, x):
            x = np.asarray(x).flatten()
            return np.vstack([np.ones_like(x), x])

    return LogLinearNoise(a=a, s=s)


def _case(name, n=300, seed=3):
    """``(gp, x, yerr, y)``: a computed dense GP for each block type."""
    import george_b200 as george
    from george_b200 import kernels as K
    rng = np.random.default_rng(seed)
    if name == "sqexp_line_loglinear":
        x = np.sort(rng.uniform(0, 10, n))
        gp = george.GP(1.3 * K.ExpSquaredKernel(0.7), mean=_line_mean(0.2, -0.1), fit_mean=True,
                       white_noise=_log_linear_noise(-3.0, 0.1), fit_white_noise=True)
    elif name == "matern_periodic_frozen":
        x = np.sort(rng.uniform(0, 10, n))
        gp = george.GP(0.8 * K.Matern32Kernel(1.5) * K.ExpSine2Kernel(gamma=2.0, log_period=0.5), mean=0.3,
                       fit_mean=True, white_noise=np.log(0.02), fit_white_noise=True)
        gp.freeze_parameter("kernel:k2:log_period")
    elif name == "rq_2d":
        x = rng.uniform(-3, 3, (n, 2))
        gp = george.GP(0.6 * K.RationalQuadraticKernel(log_alpha=np.log(0.8), metric=[1.0, 2.0], ndim=2),
                       white_noise=np.log(0.05), fit_white_noise=True)
    elif name == "co2":
        x = np.sort(rng.uniform(1958, 2003, n))
        k1 = 66 ** 2 * K.ExpSquaredKernel(metric=67 ** 2)
        k2 = 2.4 ** 2 * K.ExpSquaredKernel(90 ** 2) * K.ExpSine2Kernel(gamma=2 / 1.3 ** 2, log_period=0.0)
        k3 = 0.66 ** 2 * K.RationalQuadraticKernel(log_alpha=np.log(0.78), metric=1.2 ** 2)
        k4 = 0.18 ** 2 * K.ExpSquaredKernel(1.6 ** 2)
        gp = george.GP(k1 + k2 + k3 + k4, mean=340.0, fit_mean=True, white_noise=np.log(0.19 ** 2),
                       fit_white_noise=True)
    else:
        raise KeyError(name)
    yerr = 0.1 + 0.1 * rng.random(n)
    gp.compute(x, yerr)
    y = np.sin(x if x.ndim == 1 else x[:, 0]) + yerr * rng.standard_normal(n)
    return gp, x, yerr, y


CASES = ["sqexp_line_loglinear", "matern_periodic_frozen", "rq_2d", "co2"]
WELL_CONDITIONED = CASES[:3]  # the CO2 covariance (amplitude 66^2 over noise 0.1^2) is too ill-conditioned for 1e-10


def _cov(gp, x, yerr):
    """K(theta) in float64 from covariance values alone."""
    wn = np.asarray(gp.white_noise.get_value(x), dtype=np.float64).flatten() * np.ones(len(yerr))
    return gp.get_matrix(x) + np.diag(yerr ** 2 + np.exp(wn))


def _brute(gp, x, yerr):
    """The formula in longdouble: K^-1 by a longdouble Cholesky, dK from get_gradient, one entry at a time."""
    n = len(yerr)
    n_mean, n_wn = len(gp.mean), len(gp.white_noise)
    kinv = solve_ld(chol_ld(_cov(gp, x, yerr)), np.eye(n, dtype=LD))
    dks = []
    if n_wn:
        wn = np.asarray(gp.white_noise.get_value(x), dtype=np.float64).flatten() * np.ones(n)
        dwn = np.asarray(gp.white_noise.get_gradient(x)).reshape(n_wn, n)
        dks += [np.diag((np.exp(wn) * dwn[k]).astype(LD)) for k in range(n_wn)]
    if len(gp.kernel):
        dK = gp.kernel.get_gradient(gp.parse_samples(x)).astype(LD)
        dks += [dK[:, :, p] for p in range(dK.shape[2])]
    size = len(gp)
    F = np.zeros((size, size), dtype=LD)
    if n_mean:
        dmu = np.asarray(gp.mean.get_gradient(x), dtype=np.float64).reshape(n_mean, n).astype(LD)
        F[:n_mean, :n_mean] = dmu @ kinv @ dmu.T
    B = [kinv @ d @ kinv for d in dks]
    for a in range(len(dks)):
        for b in range(len(dks)):
            F[n_mean + a, n_mean + b] = np.sum(B[a] * dks[b]) / 2
    return F


def _rel(a, b):
    b = np.asarray(b, dtype=LD)
    return float(np.max(np.abs(np.asarray(a, dtype=LD) - b)) / np.max(np.abs(b)))


# ---- 1. brute force, 4. symmetry / PSD / repeatability ----------------------------------------------------------------
@pytest.mark.parametrize("name", WELL_CONDITIONED)
def test_dense_against_longdouble(gpu, name, record_property):
    gp, x, yerr, y = _case(name)
    F = gp.fisher_information()
    assert F.shape == (len(gp), len(gp))
    ref = _brute(gp, x, yerr)
    err = _rel(F, ref)
    record_property("rel_err", err)
    assert err < BRUTE_TOL, err
    assert np.array_equal(F, F.T)
    assert np.array_equal(F, gp.fisher_information())
    w = np.linalg.eigvalsh(F)
    assert w[0] >= -PSD_TOL * np.abs(w).max(), w


# ---- 2. Hessian of the KL divergence ----------------------------------------------------------------------------------
def test_hessian_of_kl(gpu):
    import george_b200 as george
    from george_b200 import kernels as K
    rng = np.random.default_rng(7)
    n = 120
    x = np.sort(rng.uniform(0, 8, n))
    yerr = 0.1 + 0.05 * rng.random(n)
    gp = george.GP(1.3 * K.Matern32Kernel(1.0), mean=_line_mean(0.2, -0.1), fit_mean=True,
                   white_noise=_log_linear_noise(-3.0, 0.1), fit_white_noise=True)
    gp.compute(x, yerr)
    F = gp.fisher_information()
    theta0 = gp.get_parameter_vector().copy()
    mu0 = gp.mean.get_value(x)
    K0 = _cov(gp, x, yerr)
    ld0 = 2 * np.sum(np.log(np.diag(sla.cholesky(K0, lower=True))))

    def kl(theta):
        gp.set_parameter_vector(theta)
        Kt = _cov(gp, x, yerr)
        c = sla.cho_factor(Kt, lower=True)
        d = gp.mean.get_value(x) - mu0
        ldt = 2 * np.sum(np.log(np.diag(c[0])))
        return 0.5 * (np.trace(sla.cho_solve(c, K0)) + d.dot(sla.cho_solve(c, d)) - n + ldt - ld0)

    P = len(theta0)
    h = 1e-3
    H = np.zeros((P, P))
    try:
        for a in range(P):
            ea = np.zeros(P)
            ea[a] = h
            H[a, a] = (kl(theta0 + ea) - 2 * kl(theta0) + kl(theta0 - ea)) / h ** 2
            for b in range(a):
                eb = np.zeros(P)
                eb[b] = h
                H[a, b] = H[b, a] = (kl(theta0 + ea + eb) - kl(theta0 + ea - eb) - kl(theta0 - ea + eb)
                                     + kl(theta0 - ea - eb)) / (4 * h * h)
    finally:
        gp.set_parameter_vector(theta0)
    err = float(np.max(np.abs(F - H)) / np.max(np.abs(F)))
    assert err < KL_TOL, (err, F, H)


# ---- 3. scale identity ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [300, 1025, 2049])
def test_scale_identity(gpu, n, record_property):
    import george_b200 as george
    from george_b200 import kernels as K
    rng = np.random.default_rng(n)
    x = np.sort(rng.uniform(0, 10 * n / 1000, n))
    gp = george.GP(1.7 * K.ExpSquaredKernel(0.6), white_noise=np.log(0.05), fit_white_noise=True)
    gp.compute(x, 0.0)
    F = gp.fisher_information()
    assert gp.get_parameter_names()[:2] == ("white_noise:value", "kernel:k1:log_constant")
    block = F[:2, :2].sum()
    err = abs(block - n / 2) / (n / 2)
    record_property("rel_err", err)
    assert err < SCALE_TOL, (block, n / 2)
    assert np.array_equal(F, F.T)


# ---- 5. grad bits -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("fit", ["all", "mean_only", "kernel_only"])
def test_grad_is_grad_log_likelihood(gpu, name, fit):
    gp, x, yerr, y = _case(name, n=200)
    if fit == "mean_only":
        gp.kernel.freeze_all_parameters()
        gp.white_noise.freeze_all_parameters()
    elif fit == "kernel_only":
        gp.mean.freeze_all_parameters()
        gp.white_noise.freeze_all_parameters()
    if len(gp) == 0:
        pytest.skip("nothing to fit")
    grad, F = gp.fisher_information(y)
    assert np.array_equal(grad, gp.grad_log_likelihood(y))
    assert np.array_equal(F, gp.fisher_information())


# ---- 6. host route ----------------------------------------------------------------------------------------------------
def test_host_route_against_device_route(gpu):
    from george_b200.solvers import BasicSolver

    class NoHook(BasicSolver):
        fisher_terms = None

    gp, x, yerr, y = _case("sqexp_line_loglinear", n=250)
    grad, F = gp.fisher_information(y)
    gp.solver = pickle.loads(pickle.dumps(gp.solver))  # a restored dense solver has no coordinates: host route
    assert gp.solver.fisher_terms(None, gp.kernel.unfrozen_mask, np.zeros((0, len(x)))) is None
    pgrad, pF = gp.fisher_information(y)
    assert _rel(pF, F) < HOST_TOL and _rel(pgrad, grad) < HOST_TOL
    assert np.array_equal(pF, pF.T)
    gp2, _, _, _ = _case("sqexp_line_loglinear", n=250)
    gp2.solver_type = NoHook
    gp2.compute(x, yerr)
    hgrad, hF = gp2.fisher_information(y)
    assert _rel(hF, F) < HOST_TOL and _rel(hgrad, grad) < HOST_TOL


# ---- 7. errors --------------------------------------------------------------------------------------------------------
def test_hodlr_raises(gpu):
    import george_b200 as george
    from george_b200 import kernels as K
    from george_b200.solvers import HODLRSolver
    x = np.linspace(0, 10, 500)
    gp = george.GP(1.0 * K.ExpSquaredKernel(1.0), solver=HODLRSolver, min_size=100, tol=1e-12)
    gp.compute(x, 0.1)
    with pytest.raises(NotImplementedError, match="HODLR"):
        gp.fisher_information()
    with pytest.raises(NotImplementedError, match="HODLR"):
        gp.fisher_information(np.sin(x), quiet=True)


def test_more_than_64_parameters(gpu):
    import george_b200 as george
    from george_b200 import kernels as K
    kernel = 1.0 * K.ExpSquaredKernel(np.eye(8), ndim=8)
    for _ in range(2):
        kernel = kernel + 1.0 * K.ExpSquaredKernel(np.eye(8), ndim=8)
    x = np.random.default_rng(2).uniform(-1, 1, (64, 8))
    y = np.sin(x[:, 0])
    gp = george.GP(kernel)
    gp.compute(x, 0.1)
    assert len(gp) > 64
    with pytest.raises(ValueError, match="64"):
        gp.grad_log_likelihood(y)
    with pytest.raises(ValueError, match="64"):
        gp.fisher_information()
    assert not gp.fisher_information(quiet=True).any()
    grad, F = gp.fisher_information(y, quiet=True)
    assert not grad.any() and not F.any() and F.shape == (len(gp), len(gp))
