# -*- coding: utf-8 -*-
"""Draws on the device (``bgp_mvn_sample``, ``bgp_dense_sample``, ``bgp_hodlr_sample``; GP.sample_conditional and
GP.sample with ``rng``): draws = mu + z L^T with L the lower Cholesky factor of sym(C) + jitter I.

* the factor itself, recovered exactly from an identity z, against sym(C) + jitter I in longdouble;
* random z on both product paths (rows below BGP_SAMPLE_DMMA_ROWS, DMMA from it) against longdouble, repeatability;
* the fused routes equal the generic route on predict's covariance; sample(t) and sample() routes;
* the GP contract: the generator advanced by exactly one standard_normal call, the GP untouched, rng=None unchanged,
  solvers without the hook;
* failures: a singular covariance, NaN, an indefinite HODLR covariance; one statistics check; sizes at scale.
"""
import copy

import numpy as np
import pytest

import hiprec

pytestmark = pytest.mark.gpu

LD = np.longdouble
EPS = np.finfo(np.float64).eps

# bars: 10-100x the largest value measured on one H100 80GB HBM3 (SXM, 700 W power limit); where the measured value
# is 0 the bar is a few hundred ulps of the scale
FACTOR_TOL = 5.0        # max|L L^T - A| / (ns eps max|A|), last rows          (measured 0.12; 8.0e-5 / 1.4e-4 at scale)
DRAW_TOL = 1e-16        # max|draws - ld| / (max|z| max|L| ns)                  (measured 5.1e-18)
HODLR_TOL = 1e-13       # HODLR fused vs generic above N = 1024, on the draws   (measured 0: the solve repeated its bits)
SHARD_TOL = 5e-13       # shard plug-in vs unsharded, on the draws' scale       (measured 1.6e-14)


def _lib():
    from george_b200 import _lib
    return _lib


def _mvn(cov, z, mean, jitter):
    from george_b200.utils import device_gaussian_samples
    return device_gaussian_samples(cov, z, mean, jitter)


def _sym(C):
    L = np.tril(C)
    return L + np.tril(C, -1).T


def _spd(ns, seed, cond=10.0):
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.standard_normal((ns, ns)))
    return (q * np.linspace(1.0, cond, ns)) @ q.T


def _dense_gp(n=300, seed=0, **kw):
    import george_b200 as george
    from george_b200 import kernels
    rng = np.random.default_rng(seed)
    t = np.sort(rng.uniform(0, n / 20.0, n))
    y = np.sin(t) + 0.1 * rng.standard_normal(n)
    gp = george.GP(1.0 * kernels.Matern32Kernel(1.0), **kw)
    gp.compute(t, 0.1)
    return gp, t, y


# ---- 1. the factor, recovered exactly ---------------------------------------------------------------------------

@pytest.mark.parametrize("ob", [None, "64"])
def test_identity_z_recovers_the_factor(gpu, monkeypatch, record_property, ob):
    if ob is None:
        monkeypatch.delenv("BGP_DENSE_OB", raising=False)
    else:
        monkeypatch.setenv("BGP_DENSE_OB", ob)  # every update level of the factorisation at small ns
    worst = 0.0
    for ns in (1, 2, 63, 64, 65, 127, 128, 129, 257, 1000):
        C = _spd(ns, ns)
        C[np.triu_indices(ns, 1)] += 1e-3  # an upper triangle that must not be read
        mu = np.random.default_rng(1).standard_normal(ns)
        jitter = 1e-8
        draws = _mvn(C, np.eye(ns), mu, jitter)
        Lt = draws - mu
        a, j = np.tril_indices(ns, -1)  # j < a
        assert np.array_equal(draws[a, j], mu[j])
        L = Lt.T
        A = _sym(C) + jitter * np.eye(ns)
        rows = slice(max(0, ns - 64), ns)  # the last rows see every update of the factorisation
        err = float(np.max(np.abs(L[rows].astype(LD) @ L.T.astype(LD) - A[rows].astype(LD)))
                    / (ns * EPS * np.max(np.abs(A))))
        worst = max(worst, err)
        assert err <= FACTOR_TOL, (ns, err)
    record_property("factor_err", worst)


# ---- 2. random z on both product paths --------------------------------------------------------------------------

def test_random_z_on_both_paths(gpu, record_property):
    th = _lib().BGP_SAMPLE_DMMA_ROWS
    worst = 0.0
    for ns in (100, 300):
        C = _spd(ns, 7)
        mu = np.random.default_rng(2).standard_normal(ns)
        L = hiprec.chol_ld(C.astype(LD) + LD(1e-10) * np.eye(ns, dtype=LD))
        for size in sorted({1, max(th - 1, 1), th, 129, 300}):
            z = np.random.default_rng(size).standard_normal((size, ns))
            got = _mvn(C, z, mu, 1e-10)
            again = _mvn(C, z, mu, 1e-10)
            assert np.array_equal(got, again)
            ref = mu.astype(LD) + z.astype(LD) @ L.T
            err = float(np.max(np.abs(got - ref)) / (np.max(np.abs(z)) * float(np.max(np.abs(L))) * ns))
            worst = max(worst, err)
            assert err <= DRAW_TOL, (ns, size, err)
    record_property("draw_err", worst)


# ---- 3. the routes agree ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [300, 2100])
def test_dense_fused_equals_generic(gpu, n):
    gp, t, y = _dense_gp(n)
    ts = np.linspace(t[0], t[-1], 150)
    mu, cov = gp.predict(y, ts)
    for size in (1, 20):
        z = np.random.default_rng(size).standard_normal((size, 150))
        fused = gp.solver.sample_predictive(gp.kernel, ts[:, None], mu, z, 1e-10)
        assert np.array_equal(fused, _mvn(cov, z, mu, 1e-10))


@pytest.mark.parametrize("n", [1000, 3000])
def test_hodlr_fused_equals_generic(gpu, record_property, n):
    import george_b200 as george
    gp, t, y = _dense_gp(n, solver=george.HODLRSolver, min_size=64, tol=1e-12, rng_mode="pernode")
    ts = np.linspace(t[0], t[-1], 130)
    mu, cov = gp.predict(y, ts)
    z = np.random.default_rng(3).standard_normal((20, 130))
    fused = gp.solver.sample_predictive(gp.kernel, ts[:, None], mu, z, 1e-8)
    generic = _mvn(cov, z, mu, 1e-8)
    if n <= 1024:
        assert np.array_equal(fused, generic)
    else:
        err = float(np.max(np.abs(fused - generic)) / np.max(np.abs(generic)))
        record_property("hodlr_err", err)
        assert err <= HODLR_TOL


def test_sample_routes(gpu):
    from george_b200.gp import TINY
    gp, t, y = _dense_gp(200)
    ts = np.linspace(0, 5, 70)
    g, ref = np.random.default_rng(4), np.random.default_rng(4)
    got = gp.sample(ts, 5, rng=g)
    z = ref.standard_normal((5, 70))
    want = _mvn(gp.get_matrix(ts), z, gp._call_mean(ts[:, None]), TINY)
    assert np.array_equal(got, want)
    got = gp.sample(size=3, rng=g)
    z = ref.standard_normal((3, 200))
    assert np.array_equal(got, gp.solver.apply_sqrt(z) + gp._call_mean(gp._x))
    assert gp.sample(ts, 1, rng=g).shape == (70,)


# ---- 4. the GP contract -----------------------------------------------------------------------------------------

@pytest.mark.parametrize("solver", ["basic", "hodlr"])
def test_gp_contract(gpu, solver):
    import george_b200 as george
    kw = {} if solver == "basic" else dict(solver=george.HODLRSolver, min_size=64, tol=1e-12, rng_mode="pernode")
    gp, t, y = _dense_gp(500, **kw)
    ts = np.linspace(t[0], t[-1], 90)
    mu, cov = gp.predict(y, ts)
    state = (gp.get_parameter_vector().copy(), gp.solver, gp._alpha.copy(), gp.computed)
    for g in (np.random.default_rng(11), np.random.RandomState(11)):
        ref = copy.deepcopy(g)
        draws = gp.sample_conditional(y, ts, 4, rng=g, jitter=1e-9)
        z = ref.standard_normal((4, 90))
        assert str(g.bit_generator.state if hasattr(g, "bit_generator") else g.get_state()) == \
            str(ref.bit_generator.state if hasattr(ref, "bit_generator") else ref.get_state())
        assert np.array_equal(draws, _mvn(cov, z, mu, 1e-9))
    assert gp.sample_conditional(y, ts, rng=np.random.default_rng(0)).shape == (90,)
    assert np.array_equal(state[0], gp.get_parameter_vector()) and state[1] is gp.solver
    assert np.array_equal(state[2], gp._alpha) and gp.computed == state[3]
    np.random.seed(5)
    a = gp.sample_conditional(y, ts, 2)
    np.random.seed(5)
    assert np.array_equal(a, np.random.multivariate_normal(mu, cov, 2))


def test_solvers_without_the_hook(gpu):
    import george_b200 as george
    from george_b200 import kernels

    class Plugin(george.BasicSolver):
        sample_predictive = None

    gp, t, y = _dense_gp(200, solver=Plugin)
    ts = np.linspace(0, 5, 40)
    mu, cov = gp.predict(y, ts)
    z = np.random.default_rng(1).standard_normal((3, 40))
    got = gp.sample_conditional(y, ts, 3, rng=np.random.default_rng(1))
    assert np.array_equal(got, _mvn(cov, z, mu, george.gp.TINY))
    gp = george.GP(white_noise=np.log(0.3))  # TrivialSolver: no hook, sample(t) through bgp_mvn_sample
    gp.compute(np.linspace(0, 1, 10), 0.1)
    assert getattr(gp.solver, "sample_predictive", None) is None
    ts = np.linspace(0, 1, 4)
    got = gp.sample(ts, 2, rng=np.random.default_rng(2))
    z = np.random.default_rng(2).standard_normal((2, 4))
    assert np.array_equal(got, _mvn(gp.get_matrix(ts), z, np.zeros(4), george.gp.TINY))


@pytest.mark.parametrize("P", [2])
def test_shard_plugin_agrees(gpu, record_property, P):
    import george_b200 as george
    from george_b200 import kernels
    from george_b200.solvers._hodlr import HODLRSolver as Native
    import test_gpu_hodlr_shard_predict as sp
    Native.release_parked()

    class Plugin(sp._PredictShards):
        pass

    Plugin.P = P
    n = 700
    rng = np.random.default_rng(21)
    t = np.sort(rng.uniform(0, n / 50.0, n))
    y = np.sin(t) + 0.1 * rng.standard_normal(n)
    ts = np.sort(rng.uniform(-0.5, n / 50.0 + 0.5, 90))

    def make(solver, **kw):
        gp = george.GP(1.3 * kernels.ExpKernel(1.0), solver=solver, tol=1e-12, min_size=50, exhaust="dense", **kw)
        gp.compute(t, 0.05)
        return gp

    a = make(Plugin).sample_conditional(y, ts, 5, rng=np.random.default_rng(9), jitter=1e-8)
    b = make(george.HODLRSolver, rng_mode="pernode").sample_conditional(y, ts, 5, rng=np.random.default_rng(9),
                                                                          jitter=1e-8)
    err = float(np.max(np.abs(a - b)) / np.max(np.abs(b)))
    record_property("shard_err", err)
    assert err <= SHARD_TOL
    Native.release_parked()


# ---- 5. failures ------------------------------------------------------------------------------------------------

def test_singular_and_nan_raise(gpu):
    from george_b200 import kernels
    k = 1.0 * kernels.ExpSquaredKernel(1.0)
    x = np.array([0.0, 0.0, 1.0])
    C = k.get_value(x[:, None])
    with pytest.raises(np.linalg.LinAlgError, match="2-th leading minor of the array is not positive definite"):
        _mvn(C, np.ones((2, 3)), np.zeros(3), 0.0)
    assert np.all(np.isfinite(_mvn(C, np.ones((2, 3)), np.zeros(3), 1e-6)))
    C = _spd(50, 3)
    C[20, 10] = np.nan
    with pytest.raises(np.linalg.LinAlgError):
        _mvn(C, np.ones((1, 50)), np.zeros(50), 1e-6)
    C[20, 10] = C[10, 20] = 0.0
    C[30, 30] = np.nan
    with pytest.raises(np.linalg.LinAlgError, match="31-th"):
        _mvn(C, np.ones((9, 50)), np.zeros(50), 1e-6)


def test_noise_free_conditional_with_zero_jitter(gpu):
    import george_b200 as george
    from george_b200 import kernels
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0))
    gp.compute(np.linspace(0, 3, 10), 1e-3)
    ts = np.array([5.0, 5.0, 6.0])
    with pytest.raises(np.linalg.LinAlgError, match="2-th leading minor"):
        gp.sample_conditional(np.zeros(10), ts, rng=np.random.default_rng(0), jitter=0.0)
    assert gp.sample_conditional(np.zeros(10), ts, rng=np.random.default_rng(0), jitter=1e-6).shape == (3,)


def test_indefinite_hodlr_covariance_raises_and_gp_survives(gpu):
    import george_b200 as george
    from george_b200 import kernels
    rng = np.random.default_rng(5)
    n = 2000
    t = np.sort(rng.uniform(0, 10, n))
    y = np.sin(t)
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(0.5), solver=george.HODLRSolver, min_size=50)  # tol = 0.1
    gp.compute(t, 1e-3)
    ts = np.linspace(0, 10, 400)
    mu, cov = gp.predict(y, ts)
    if np.all(np.linalg.eigvalsh(_sym(cov)) > 0):
        pytest.skip("this factorisation's predictive covariance is positive definite")
    with pytest.raises(np.linalg.LinAlgError, match="jitter"):
        gp.sample_conditional(y, ts, rng=np.random.default_rng(0), jitter=0.0)
    mu2, cov2 = gp.predict(y, ts)
    assert np.array_equal(mu, mu2) and np.array_equal(cov, cov2)


# ---- 6. statistics ----------------------------------------------------------------------------------------------

def test_sample_covariance(gpu):
    C = np.array([[2.0, 0.5, -0.3], [0.5, 1.0, 0.2], [-0.3, 0.2, 0.7]])
    size = 200000
    z = np.random.default_rng(8).standard_normal((size, 3))
    d = _mvn(C, z, np.array([1.0, -2.0, 0.5]), 0.0)
    S = np.cov(d.T)
    sigma = np.sqrt((C ** 2 + np.outer(np.diag(C), np.diag(C))) / size)  # std of a Wishart entry / size
    assert np.all(np.abs(S - C) <= 5 * sigma)
    assert np.all(np.abs(d.mean(axis=0) - [1.0, -2.0, 0.5]) <= 5 * np.sqrt(np.diag(C) / size))


# ---- 7. at scale ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", ["dense", "hodlr"])
def test_at_scale(gpu, record_property, case):
    import george_b200 as george
    if case == "dense":
        gp, t, y = _dense_gp(8192)
        ns, size, jitter = 4096, 256, 1e-8
    else:
        gp, t, y = _dense_gp(1 << 17, solver=george.HODLRSolver, min_size=256, tol=1e-10, exhaust="lowrank")
        ns, size, jitter = 2048, 64, 1e-8
    ts = np.sort(np.random.default_rng(1).uniform(t[0], t[-1], ns))
    mu, cov = gp.predict(y, ts)
    z = np.random.default_rng(2).standard_normal((size, ns))
    fused = gp.solver.sample_predictive(gp.kernel, ts[:, None], mu, z, jitter)
    generic = _mvn(cov, z, mu, jitter)
    if case == "dense":
        assert np.array_equal(fused, generic)
    else:
        err = float(np.max(np.abs(fused - generic)) / np.max(np.abs(generic)))
        record_property("hodlr_scale_err", err)
        assert err <= HODLR_TOL
    # backward error of L from an identity z, on a block of rows: (L L^T)[r, :] vs A[r, :]
    Lt = _mvn(cov, np.eye(ns), np.zeros(ns), jitter)
    L = Lt.T
    A = _sym(cov) + jitter * np.eye(ns)
    rows = slice(ns - 32, ns)
    err = float(np.max(np.abs(L[rows].astype(LD) @ L.T.astype(LD) - A[rows].astype(LD)))
                / (ns * EPS * np.max(np.abs(A))))
    record_property("scale_factor_err_" + case, err)
    assert err <= FACTOR_TOL
