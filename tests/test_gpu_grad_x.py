# -*- coding: utf-8 -*-
"""``GP.grad_log_likelihood_x``, the log-likelihood gradient with respect to the training inputs, on the device
(``bgp_dense_grad_x_terms``, ``bgp_hodlr_grad_x_terms``, ``bgp_hodlr_grad_x_terms_local_dev``):

1. dense against a longdouble brute force with analytic dk/dx (the radial kernels, every metric form) and against
   central differences of ``log_likelihood`` in x over the kernel zoo; dimensions outside a kernel's axes give zeros;
2. ``grad``, ``alpha`` and ``diagA`` are ``grad_log_likelihood``'s bits on dense, HODLR resident and HODLR streamed;
3. HODLR on exact trees against dense, ``dx`` bit-identical across slab widths and repeated calls, resident against
   streamed;
4. translation invariance of a stationary kernel: ``sum_i dx_i = 0`` to rounding;
5. host-exchange shards on one device against the unsharded handle, rows outside a shard left alone, P = 1 against the
   streamed entry bit for bit;
6. the host route (a plug-in without the hook, a pickled dense solver) against the device route;
7. a time delay fitted through the chain rule against a central difference;
8. the error returns.
"""
import pickle

import numpy as np
import pytest

import test_gpu_hodlr_grad_stream as gs
import test_gpu_hodlr_shards as sh
from conftest import make_kernels

pytestmark = pytest.mark.gpu

LD = np.longdouble
BGP_ERR_INVALID, BGP_ERR_NOT_COMPUTED = 1, 3
SENTINEL = -321.5

BRUTE_TOL = 1e-10   # dense dx vs longdouble, relative to max |dx|
FD_TOL = 2e-5       # dense dx vs central differences of log_likelihood, relative to max |dx|
EXACT_TOL = 1e-8    # HODLR (tol 1e-12) vs dense, relative to max |dx|
MODE_TOL = 1e-11    # HODLR resident vs streamed, relative to max |dx|
SHIFT_TOL = 1e-12   # |sum_i dx_i| / sum_i |dx_i|                     (measured 1.7e-15, HODLR streamed)
SHARD_TOL = 1e-9    # assembled shards vs the unsharded handle, relative to max |dx|


@pytest.fixture
def clean(monkeypatch):
    from george_b200.solvers._hodlr import HODLRSolver
    for var in ("BGP_GRAD_CHUNK", "BGP_PREDICT_CHUNK"):
        monkeypatch.delenv(var, raising=False)
    HODLRSolver.release_parked()
    yield monkeypatch
    HODLRSolver.release_parked()


def _lib():
    from george_b200 import _lib
    return _lib


def _rel(a, b):
    return float(np.max(np.abs(np.asarray(a, dtype=LD) - np.asarray(b, dtype=LD))) / max(np.max(np.abs(b)), 1e-300))


def _data(n, nd=1, seed=11, span=None):
    rng = np.random.default_rng(seed)
    span = span or 0.02 * n
    x = rng.uniform(0, span, (n, nd))
    if nd == 1:
        x = np.sort(x[:, 0])[:, None]
    yerr = 0.1 + 0.05 * rng.random(n)
    y = np.sin(x[:, 0]) + 0.2 * rng.standard_normal(n)
    return x, yerr, y


def _gp(kernel, x, yerr, solver=None, **kwargs):
    import george_b200 as george
    gp = george.GP(kernel, mean=0.1, fit_mean=True, white_noise=np.log(0.01), fit_white_noise=True, solver=solver,
                   **kwargs)
    gp.compute(x, yerr)
    return gp


# ---- 1. dense against longdouble and finite differences -------------------------------------------------------------

_PROFILES = {  # (kernel class, dk/dr2 of the profile in longdouble)
    "expsq": ("ExpSquaredKernel", lambda r2: -0.5 * np.exp(-0.5 * r2)),
    "m32": ("Matern32Kernel", lambda r2: -1.5 * np.exp(-np.sqrt(3 * r2))),
    "m52": ("Matern52Kernel", lambda r2: -5.0 / 6.0 * (1 + np.sqrt(5 * r2)) * np.exp(-np.sqrt(5 * r2))),
    "exp": ("ExpKernel", lambda r2: np.where(r2 > 0, -0.5 * np.exp(-np.sqrt(r2)) / np.sqrt(np.where(r2 > 0, r2, 1)), 0)),
}
_METRICS = {
    "iso": (0.8, lambda: np.eye(3) * 0.8),
    "axis": ([0.5, 1.0, 2.0], lambda: np.diag([0.5, 1.0, 2.0])),
    "general": ([[1.0, 0.1, 0.2], [0.1, 2.0, 0.3], [0.2, 0.3, 1.5]],
                lambda: np.array([[1.0, 0.1, 0.2], [0.1, 2.0, 0.3], [0.2, 0.3, 1.5]])),
}


def _brute_dx(profile, M, c, x, yerr, wn, y, mu, value):
    """dx in longdouble for k = c f(r2), r2 = d^T M^-1 d, K = k(x, x) + diag(yerr^2 + exp(wn))."""
    xl = np.asarray(x, dtype=LD)
    Minv = np.linalg.inv(np.asarray(M, dtype=np.float64)).astype(LD)
    d = xl[:, None, :] - xl[None, :, :]
    Md = np.einsum("pq,ijq->ijp", Minv, d)
    r2 = np.einsum("ijq,ijq->ij", d, Md)
    K = c * value(r2) + np.diag(np.asarray(yerr, dtype=LD) ** 2 + LD(np.exp(wn)))
    Kinv = np.linalg.inv(K.astype(np.float64)).astype(LD)  # refined once below in longdouble
    Kinv = Kinv + Kinv.dot(np.eye(len(x), dtype=LD) - K.dot(Kinv))
    alpha = Kinv.dot(np.asarray(y, dtype=LD) - LD(mu))
    A = np.outer(alpha, alpha) - Kinv
    fp = c * profile(r2)
    return np.einsum("ij,ij,ijq->iq", A, 2 * fp, Md)


_VALUES = {
    "expsq": lambda r2: np.exp(-0.5 * r2),
    "m32": lambda r2: (1 + np.sqrt(3 * r2)) * np.exp(-np.sqrt(3 * r2)),
    "m52": lambda r2: (1 + np.sqrt(5 * r2) + 5 * r2 / 3) * np.exp(-np.sqrt(5 * r2)),
    "exp": lambda r2: np.exp(-np.sqrt(r2)),
}


@pytest.mark.parametrize("metric", sorted(_METRICS))
@pytest.mark.parametrize("name", sorted(_PROFILES))
def test_dense_against_longdouble(gpu, name, metric):
    from george_b200 import kernels as K
    cls, profile = _PROFILES[name]
    m, M = _METRICS[metric]
    x, yerr, y = _data(300, nd=3, span=4.0)
    gp = _gp(1.7 * getattr(K, cls)(m, ndim=3), x, yerr)
    dx = gp.grad_log_likelihood_x(y)
    ref = _brute_dx(profile, M(), 1.7, x, yerr, np.log(0.01), y, 0.1, _VALUES[name])
    assert dx.shape == (300, 3)
    assert _rel(dx, ref) < BRUTE_TOL


def _fd_zoo():
    from george_b200 import kernels as K
    zoo = [(n, k) for n, k in make_kernels() if n not in ("expsq_block", "empty")]
    zoo += [("dot_1d", K.DotProductKernel() + 1.0 * K.ExpSquaredKernel(1.0)),
            ("cauchy_x_damped", K.CauchyKernel(metric=1.5, ndim=2) * K.DampedCosineKernel(
                log_period=np.log(3.0), log_decay=0.2, ndim=2, axes=1) + 0.5 * K.Matern32Kernel(1.0, ndim=2))]
    return zoo


@pytest.mark.parametrize("name,kernel", _fd_zoo(), ids=[z[0] for z in _fd_zoo()])
def test_dense_against_finite_differences(gpu, name, kernel):
    nd = kernel.ndim
    x, yerr, y = _data(60, nd=nd, seed=3, span=3.0)
    x = x + 0.5  # away from 0: Linear / Polynomial of x1 * x2 at non-integer powers
    gp = _gp(kernel, x, yerr)
    dx = gp.grad_log_likelihood_x(y)
    fd = np.zeros_like(dx)
    for i in range(len(x)):
        for q in range(nd):
            h = 1e-6 * max(1.0, abs(x[i, q]))
            vals = []
            for sgn in (1, -1):
                xp = x.copy()
                xp[i, q] += sgn * h
                gp.compute(xp, yerr)
                vals.append(gp.log_likelihood(y))
            fd[i, q] = (vals[0] - vals[1]) / (2 * h)
    assert _rel(dx, fd) < FD_TOL, name


def test_dimensions_outside_the_axes_are_zero(gpu):
    from george_b200 import kernels as K
    x, yerr, y = _data(200, nd=3, span=4.0)
    gp = _gp(K.Matern32Kernel(1.0, ndim=3, axes=[0, 2]) + K.CosineKernel(log_period=0.3, ndim=3, axes=0), x, yerr)
    dx = gp.grad_log_likelihood_x(y)
    assert np.all(dx[:, 1] == 0.0) and np.all(dx[:, 0] != 0.0)


# ---- 2-4. HODLR and the bits of grad_log_likelihood -----------------------------------------------------------------

def _hodlr_gp(x, yerr, tol=1e-12, kernel=None):
    from george_b200 import kernels as K
    from george_b200.solvers import HODLRSolver
    return _gp(kernel or 1.3 * K.Matern32Kernel(0.9), x, yerr, solver=HODLRSolver, min_size=64, tol=tol,
               rng_mode="pernode")


@pytest.mark.parametrize("mode", ["dense", "resident", "streamed"])
def test_return_gradient_is_grad_log_likelihood(gpu, clean, mode):
    from george_b200 import kernels as K
    x, yerr, y = _data(1001)
    if mode == "streamed":
        clean.setenv("BGP_GRAD_CHUNK", "128")
    k = 1.3 * K.Matern32Kernel(0.9)
    gp = _gp(k, x, yerr) if mode == "dense" else _hodlr_gp(x, yerr, kernel=k)
    gp.freeze_parameter("white_noise:value")
    grad, dx = gp.grad_log_likelihood_x(y, return_gradient=True)
    assert np.array_equal(grad, gp.grad_log_likelihood(y))
    which = gp.kernel.unfrozen_mask.astype(np.uint32)
    r = gp._residual(y)
    a1, g1, d1 = gp.solver.grad_terms(r, which)
    a2, g2, d2, dx2 = gp.solver.grad_x_terms(r, which)
    assert np.array_equal(a1, a2) and np.array_equal(g1, g2) and np.array_equal(d1, d2)
    assert np.array_equal(dx2, dx)
    assert np.array_equal(gp.solver.grad_x_terms(r, None)[3], dx)  # the parameter contraction does not touch dx


def test_hodlr_against_dense_and_across_slabs(gpu, clean):
    from george_b200 import kernels as K
    k = 1.3 * K.Matern32Kernel(0.9)
    x, yerr, y = _data(1001)
    ref = _gp(k, x, yerr).grad_log_likelihood_x(y)
    gp = _hodlr_gp(x, yerr, kernel=k)
    resident = gp.grad_log_likelihood_x(y)
    assert _rel(resident, ref) < EXACT_TOL
    streamed = []
    for c in ("64", "128", "192"):
        clean.setenv("BGP_GRAD_CHUNK", c)
        streamed.append(gp.grad_log_likelihood_x(y))
    streamed.append(gp.grad_log_likelihood_x(y))
    for s in streamed[1:]:
        assert np.array_equal(s, streamed[0])
    assert _rel(streamed[0], resident) < MODE_TOL
    assert _rel(streamed[0], ref) < EXACT_TOL


@pytest.mark.parametrize("mode", ["dense", "resident", "streamed"])
def test_translation_invariance(gpu, clean, record_property, mode):
    from george_b200 import kernels as K
    x, yerr, y = _data(700, nd=2, span=6.0)
    if mode == "streamed":
        clean.setenv("BGP_GRAD_CHUNK", "192")
    k = 1.1 * K.ExpSquaredKernel([0.6, 1.4], ndim=2)
    gp = _gp(k, x, yerr) if mode == "dense" else _hodlr_gp(x, yerr, kernel=k)
    dx = gp.grad_log_likelihood_x(y)
    shift = np.abs(dx.sum(axis=0)) / np.abs(dx).sum(axis=0)
    record_property("shift", float(shift.max()))
    assert np.all(shift <= SHIFT_TOL)


def test_non_stationary_streamed_against_dense(gpu, clean):
    from george_b200 import kernels as K
    k = 0.5 * K.DotProductKernel() + 1.0 * K.Matern52Kernel(0.8)
    x, yerr, y = _data(600, seed=4)
    ref = _gp(k, x, yerr).grad_log_likelihood_x(y)
    clean.setenv("BGP_GRAD_CHUNK", "64")
    gp = _hodlr_gp(x, yerr, kernel=k, tol=1e-13)
    assert _rel(gp.grad_log_likelihood_x(y), ref) < EXACT_TOL


# ---- 5. host-exchange shards ----------------------------------------------------------------------------------------

def _local_x(s, alpha, which, n, nd):
    a = sh._Dev(n)
    a.upload(alpha)
    dx = sh._Dev(n * nd)
    dx.upload(np.full(n * nd, SENTINEL))
    g = s.grad_x_terms_local(a.p, which, dx.p)
    return g, dx.download().reshape(n, nd)


@pytest.mark.parametrize("P", [1, 2, 4])
def test_shards_against_the_unsharded_handle(gpu, clean, P):
    from george_b200 import kernels as K
    kernel = 1.3 * K.Matern32Kernel(0.9, ndim=2)
    n, nd = 3000, 2
    x, yerr, y = _data(n, nd=nd, span=40.0)
    opts = dict(min_size=64, tol=1e-12)
    single = sh._single(kernel, x, yerr, **opts)
    which = np.ones(2, dtype=np.uint32)
    alpha, g, diag, dx = (np.empty(n), np.zeros(2), np.empty(n), np.empty((n, nd)))
    clean.setenv("BGP_GRAD_CHUNK", "256")
    _lib().check(single._lib.bgp_hodlr_grad_x_terms(single._ptr, _lib().ptr(which), _lib().ptr(y), _lib().ptr(alpha),
                                                    _lib().ptr(g), _lib().ptr(diag), _lib().ptr(dx)))
    if P == 1:
        g1, dx1 = _local_x(single, alpha, which, n, nd)
        assert np.array_equal(g1, g) and np.array_equal(dx1, dx)
        return
    shards = sh._shards(kernel, x, yerr, P, **opts)
    alphas = [o[:, 0].copy() for o in sh._sharded_solve(shards, y[:, None])]
    assembled = np.full((n, nd), np.nan)
    gsum = np.zeros(2)
    for s, (row0, rows), a in zip(shards.handles, shards.ranges, alphas):
        gp_, d = _local_x(s, a, which, n, nd)
        outside = np.r_[d[:row0], d[row0 + rows:]]
        assert np.all(outside == SENTINEL), "a shard wrote dx rows outside its slice"
        assembled[row0:row0 + rows] = d[row0:row0 + rows]
        gsum += gp_
    assert _rel(assembled, dx) < SHARD_TOL
    assert np.max(np.abs(gsum - g) / np.abs(g)) < SHARD_TOL


def _dev_of(a, count):
    d = sh._Dev(count)
    d.upload(np.ascontiguousarray(a, dtype=np.float64))
    return d


# ---- 6. host route --------------------------------------------------------------------------------------------------

def test_host_route_against_device_route(gpu):
    from george_b200 import kernels as K
    from george_b200.solvers import BasicSolver

    class NoHook(BasicSolver):
        grad_x_terms = None
        grad_terms = None

    k = 1.3 * K.Matern52Kernel(0.9, ndim=2)
    x, yerr, y = _data(400, nd=2, span=8.0)
    gp = _gp(k, x, yerr)
    grad, dx = gp.grad_log_likelihood_x(y, return_gradient=True)
    host = _gp(k, x, yerr, solver=NoHook)
    hgrad, hdx = host.grad_log_likelihood_x(y, return_gradient=True)
    assert np.array_equal(hgrad, host.grad_log_likelihood(y))
    assert _rel(hdx, dx) < MODE_TOL and _rel(hgrad, grad) < MODE_TOL
    gp.solver = pickle.loads(pickle.dumps(gp.solver))  # a restored dense solver has no coordinates: host route
    assert gp.solver.grad_x_terms(gp._residual(y), None) is None
    pgrad, pdx = gp.grad_log_likelihood_x(y, return_gradient=True)
    assert _rel(pdx, dx) < MODE_TOL and _rel(pgrad, grad) < MODE_TOL


# ---- 7. time delay --------------------------------------------------------------------------------------------------

def test_time_delay_chain_rule(gpu):
    import george_b200 as george
    from george_b200 import kernels as K
    rng = np.random.default_rng(2)
    t1, t2 = np.sort(rng.uniform(0, 20, 80)), np.sort(rng.uniform(0, 20, 70))
    yerr = 0.05 * np.ones(150)
    y = np.r_[np.sin(t1), np.sin(t2 - 1.3)] + 0.05 * rng.standard_normal(150)
    gp = george.GP(0.8 * K.Matern32Kernel(2.0))

    def ll(delta):
        gp.compute(np.r_[t1, t2 - delta], yerr)
        return gp.log_likelihood(y)

    delta = 1.1
    gp.compute(np.r_[t1, t2 - delta], yerr)
    g, dx = gp.grad_log_likelihood_x(y, return_gradient=True)
    ddelta = -dx[len(t1):, 0].sum()
    h = 1e-5
    fd = (ll(delta + h) - ll(delta - h)) / (2 * h)
    assert abs(ddelta - fd) < 1e-5 * max(1.0, abs(fd))


# ---- 8. errors ------------------------------------------------------------------------------------------------------

def test_error_returns(gpu, clean):
    from george_b200 import kernels as K
    from george_b200.solvers import BasicSolver
    lib = _lib().load()
    n = 200
    # more than 8 input dimensions
    x9, yerr, y = _data(n, nd=9, span=5.0)
    k9 = K.ExpSquaredKernel(1.0, ndim=9, axes=[0, 1])  # nine input dimensions; a kernel may act on at most 8 axes
    s = BasicSolver(k9)
    s.compute(x9, yerr)
    out = [np.empty(n), np.zeros(2), np.empty(n), np.empty(n * 9)]
    w = np.ones(2, dtype=np.uint32)
    assert lib.bgp_dense_grad_x_terms(s._handle.ptr, _lib().ptr(w), _lib().ptr(y), *[_lib().ptr(o) for o in out]) \
        == BGP_ERR_INVALID
    assert "at most 8 dimensions" in _lib().last_error()
    h9 = sh._single(k9, x9, yerr, min_size=64, tol=1e-10)
    assert lib.bgp_hodlr_grad_x_terms(h9._ptr, _lib().ptr(w), _lib().ptr(y), *[_lib().ptr(o) for o in out]) \
        == BGP_ERR_INVALID
    a = _dev_of(np.ones(n), n)
    d = _dev_of(np.zeros(n * 9), n * 9)
    assert lib.bgp_hodlr_grad_x_terms_local_dev(h9._ptr, _lib().ptr(w), a.p, None, None, d.p) == BGP_ERR_INVALID
    # more than 64 kernel parameters with a non-NULL which; NULL which skips the check
    big = gs._ksum([K.Matern32Kernel([1.0] * 8, ndim=8) for _ in range(8)] + [K.ConstantKernel(log_constant=0.1, ndim=8)])
    assert len(big) == 65
    x, yerr, y = _data(n, nd=8, span=5.0)
    s = BasicSolver(big)
    s.compute(x, yerr)
    w65 = np.ones(65, dtype=np.uint32)
    out = [np.empty(n), np.zeros(65), np.empty(n), np.empty(n * 8)]
    assert lib.bgp_dense_grad_x_terms(s._handle.ptr, _lib().ptr(w65), _lib().ptr(y), *[_lib().ptr(o) for o in out]) \
        == BGP_ERR_INVALID
    assert lib.bgp_dense_grad_x_terms(s._handle.ptr, None, _lib().ptr(y), _lib().ptr(out[0]), None,
                                      _lib().ptr(out[2]), _lib().ptr(out[3])) == 0
    hb = sh._single(big, x, yerr, min_size=64, tol=1e-10)
    assert lib.bgp_hodlr_grad_x_terms(hb._ptr, _lib().ptr(w65), _lib().ptr(y), *[_lib().ptr(o) for o in out]) \
        == BGP_ERR_INVALID
    a1, d1 = _dev_of(np.ones(n), n), _dev_of(np.zeros(n * 8), n * 8)
    assert lib.bgp_hodlr_grad_x_terms_local_dev(hb._ptr, _lib().ptr(w65), a1.p, None, None, d1.p) == BGP_ERR_INVALID
    # not computed
    from george_b200.solvers._hodlr import HODLRSolver
    fresh = sh._native()
    assert lib.bgp_hodlr_grad_x_terms(fresh._ptr, None, _lib().ptr(y), None, None, None, _lib().ptr(out[3])) == \
        BGP_ERR_NOT_COMPUTED
    assert lib.bgp_hodlr_grad_x_terms_local_dev(fresh._ptr, None, a1.p, None, None, d1.p) == BGP_ERR_NOT_COMPUTED
    del fresh
    HODLRSolver.release_parked()
    # a NULL alpha_dev / dx_dev
    x, yerr, y = _data(n)
    h1 = sh._single(1.0 * K.Matern32Kernel(1.0), x, yerr, min_size=64, tol=1e-10)
    assert lib.bgp_hodlr_grad_x_terms_local_dev(h1._ptr, None, None, None, None, d1.p) == BGP_ERR_INVALID
    assert "alpha_dev is null" in _lib().last_error()
    assert lib.bgp_hodlr_grad_x_terms_local_dev(h1._ptr, None, a1.p, None, None, None) == BGP_ERR_INVALID
    # a host-exchange shard
    xs, yerrs, ys = _data(2000, span=40.0)
    shards = sh._shards(1.0 * K.Matern32Kernel(1.0), xs, yerrs, 2, min_size=64, tol=1e-10)
    o = np.empty(2000)
    assert lib.bgp_hodlr_grad_x_terms(shards.handles[0]._ptr, None, _lib().ptr(ys), None, None, None, _lib().ptr(o)) \
        == BGP_ERR_INVALID
    assert _lib().last_error() == "grad_x_terms is not available on a sharded factorisation"
