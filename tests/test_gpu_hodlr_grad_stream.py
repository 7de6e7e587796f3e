# -*- coding: utf-8 -*-
"""``bgp_hodlr_grad_terms`` with K^-1 streamed in column slabs (csrc/hodlr.cu, csrc/kmat_ops.cu).

Above n = 65536 (or with ``BGP_GRAD_CHUNK`` set) the gradient never holds K^-1: each slab W = K^-1 E_J of identity
columns J is solved with the row-restricted solve (only the leaves and nodes meeting the rows J run) and contracted over
every ordered pair (i, j in J).  The checks:

* accuracy against a longdouble K^-1 and the oracle's gradient tensor on exact-K trees (``ExpKernel`` on sorted 1-D
  inputs, ``exhaust="dense"``: the HODLR matrix IS K), over slab widths, ragged tails, both rng modes, the big-rank level
  path, frozen parameters, 1 to 64 parameters and a generated user kernel;
* the restricted solve is the unrestricted one, bit for bit, where the solve has no atomics (n <= 1024);
* g and diag do not depend on the slab width, and two calls agree bit for bit;
* ``GP.grad_log_likelihood`` with a fitted mean model and a fitted non-constant white-noise model;
* N = 2^17 on the default selection, where the resident K^-1 (128 GiB) cannot be formed;
* the error returns, with and without ``BGP_GRAD_CHUNK``.
"""

import functools
import operator

import numpy as np
import pytest

import hiprec

pytestmark = pytest.mark.gpu

LD = np.longdouble

# bars: 10-60x the largest value measured on one H100 80GB HBM3 (SXM, 700 W power limit)
GRAD_TOL = 2e-10          # alpha, diag (relative 2-norm) and g / sum |dK| |A| vs longdouble, exact K (measured 6.4e-12)
BIG_RANK_TOL = 5e-10      # the same with every level on the big-rank path                         (measured 1.5e-11)
GRAD_TOL_LAPACK = 1e-10   # the same at n = 4097 against LAPACK's float64 K^-1                     (measured 2.2e-12)
OWN_INV_TOL = 3e-13       # g / scale and diag vs the HODLR's own K^-1 (get_inverse) in longdouble  (measured 1.1e-14)
RESIDENT_TOL = 5e-15      # g / scale, streamed vs resident (only the summation order differs)      (measured 1.6e-16)
GP_TOL = 2e-14            # GP gradient vs longdouble, relative to sum |terms| per entry           (measured 4.4e-16)
FULL_IDENTITY_TOL = 3e-15  # N = 2^17: |g_logA - identity| / sum |identity terms|                  (measured 5.7e-17)
FULL_FD_TOL = 5e-8        # N = 2^17: |grad - centred difference| / max(1, |grad|)                 (measured 1.5e-9)

BGP_OK, BGP_ERR_INVALID, BGP_ERR_NOT_COMPUTED = 0, 1, 3

SIZES = [(1, 1), (63, 16), (64, 16), (65, 16), (257, 32), (700, 50), (1025, 64), (4097, 128)]
CHUNKS = ["64", "128", "192"]
LD_MAX_N = 1100  # longdouble K^-1 up to here, LAPACK above


@pytest.fixture
def env(monkeypatch):
    for var in ("BGP_GRAD_CHUNK", "BGP_SMALL_RANK_LIMIT", "BGP_LEAF_COLS", "BGP_NO_GRAPH", "BGP_NO_CULL",
                "BGP_LEAF_FACTOR", "BGP_PREDICT_CHUNK"):
        monkeypatch.delenv(var, raising=False)
    return monkeypatch


def _solver(kernel, min_size, rng_mode="pernode", exhaust="dense", tol=1e-12):
    import george_b200 as george
    return george.HODLRSolver(kernel, min_size=min_size, tol=tol, seed=42, rng_mode=rng_mode, exhaust=exhaust)


def _exp_inputs(n, seed=0):
    rng = np.random.default_rng(seed + n)
    x = np.sort(rng.uniform(0, n / 50.0, n))[:, None]
    return x, 0.1 * np.ones(n)


_KINV = {}


def _exact_kinv(kernel, x, yerr, key):
    """K^-1 of the dense K = kernel(x) + diag(yerr^2): longdouble LDL^T up to LD_MAX_N, LAPACK above."""
    if key not in _KINV:
        n = x.shape[0]
        K = kernel.get_value(x)
        K[np.diag_indices(n)] += yerr ** 2
        if n <= LD_MAX_N:
            L, d = hiprec.ldlt_ld(K)
            _KINV[key] = (hiprec.solve_ld(L * np.sqrt(d)[None, :], np.eye(n)), True)
        else:
            import scipy.linalg
            _KINV[key] = (scipy.linalg.cho_solve(scipy.linalg.cho_factor(K, lower=True), np.eye(n)).astype(LD), False)
    return _KINV[key]


def _rel(X, Xr):
    Xr = np.asarray(Xr, dtype=LD)
    den = np.sum(Xr ** 2)
    return float(np.sqrt(np.sum((np.asarray(X, dtype=LD) - Xr) ** 2) / (den if den > 0 else 1)))


def _grad_errors(kernel, x, Kinv, r, which, alpha, g, diag):
    """alpha, g (scaled by sum |dK| |A|, per parameter) and diag against the terms built from Kinv in longdouble."""
    Kinv = np.asarray(Kinv, dtype=LD)
    alpha_ref = Kinv @ r.astype(LD)
    A = np.outer(alpha_ref, alpha_ref) - Kinv
    dK = kernel.get_gradient(x, include_frozen=True).astype(LD)
    dK[:, :, np.asarray(which) == 0] = 0
    g_ref = np.einsum("ijk,ij->k", dK, A)
    scale = np.einsum("ijk,ij->k", np.abs(dK), np.abs(A))
    scale[scale == 0] = 1
    return {"alpha": _rel(alpha, alpha_ref), "g": float(np.max(np.abs(g - g_ref) / scale)),
            "diag": _rel(diag, np.diag(A))}


def _rhs(x):
    return np.sin(3.0 * x[:, 0]) + 0.5


def _streamed(s, r, which, env, chunk):
    env.setenv("BGP_GRAD_CHUNK", chunk)
    out = s.grad_terms(r, which)
    t = s.solver.grad_timing()
    n = len(r)
    c = min((int(chunk) + 63) // 64 * 64, (n + 63) // 64 * 64)
    assert t["slab_cols"] == c and t["slabs"] == -(-n // c), t
    env.delenv("BGP_GRAD_CHUNK")
    return out


def _resident(s, r, which):
    out = s.grad_terms(r, which)
    assert s.solver.grad_timing()["slabs"] == 0
    return out


# ---- 1. accuracy of the streamed path ---------------------------------------------------------------------------

@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("rng_mode", ["pernode", "reference"])
@pytest.mark.parametrize("n,min_size", SIZES)
def test_streamed_against_longdouble(gpu, env, record_property, n, min_size, rng_mode, chunk):
    from george_b200 import kernels as K
    kernel = 1.0 * K.ExpKernel(1.0)
    x, yerr = _exp_inputs(n)
    s = _solver(kernel, min_size, rng_mode)
    s.compute(x, yerr)
    Kinv, exact = _exact_kinv(kernel, x, yerr, ("exp", n))
    r = _rhs(x)
    which = np.ones(len(kernel.get_parameter_vector(include_frozen=True)), dtype=np.uint32)
    errs = _grad_errors(kernel, x, Kinv, r, which, *_streamed(s, r, which, env, chunk))
    record_property("grad_err", max(errs.values()))
    assert max(errs.values()) <= (GRAD_TOL if exact else GRAD_TOL_LAPACK), errs


@pytest.mark.parametrize("chunk", ["64", "192"])
@pytest.mark.parametrize("n,min_size", [(66, 33), (257, 32), (700, 50), (1025, 64)])
def test_streamed_big_rank_levels(gpu, env, record_property, n, min_size, chunk):
    """BGP_SMALL_RANK_LIMIT=0: every level takes launch_level_big, whose Gram, LU and update descriptors are then
    built for the restricted node range only."""
    from george_b200 import kernels as K
    env.setenv("BGP_SMALL_RANK_LIMIT", "0")
    kernel = 1.0 * K.ExpKernel(1.0)
    x, yerr = _exp_inputs(n)
    s = _solver(kernel, min_size)
    s.compute(x, yerr)
    Kinv, _ = _exact_kinv(kernel, x, yerr, ("exp", n))
    r = _rhs(x)
    which = np.ones(2, dtype=np.uint32)
    errs = _grad_errors(kernel, x, Kinv, r, which, *_streamed(s, r, which, env, chunk))
    record_property("grad_err", max(errs.values()))
    assert max(errs.values()) <= BIG_RANK_TOL, errs


def test_streamed_frozen_parameter(gpu, env, record_property):
    """A parameter with which = 0 gets exactly 0; the others are unaffected."""
    from george_b200 import kernels as K
    kernel = 1.0 * K.ExpKernel(1.0)
    n = 700
    x, yerr = _exp_inputs(n)
    s = _solver(kernel, 50)
    s.compute(x, yerr)
    Kinv, _ = _exact_kinv(kernel, x, yerr, ("exp", n))
    r = _rhs(x)
    for which in ([0, 1], [1, 0]):
        which = np.asarray(which, dtype=np.uint32)
        alpha, g, diag = _streamed(s, r, which, env, "128")
        assert np.all(g[which == 0] == 0.0)
        errs = _grad_errors(kernel, x, Kinv, r, which, alpha, g, diag)
        record_property("grad_err", max(errs.values()))
        assert max(errs.values()) <= GRAD_TOL, errs


def _ksum(ks):
    return functools.reduce(operator.add, ks)


def _param_kernels():
    """(name, kernel, ndim, P): both NPMAX instantiations of the slab contraction and a generated user kernel."""
    from george_b200 import kernels as K
    m8 = [0.5 + 0.1 * i for i in range(8)]
    four = [(0.5 + 0.2 * i) * K.Matern32Kernel(0.6 + 0.3 * i) for i in range(4)]
    return [
        ("p1", K.ExpKernel(1.0), 1, 1),
        ("p8", _ksum(four), 1, 8),
        ("p9", _ksum(four + [K.ConstantKernel(log_constant=0.1)]), 1, 9),
        ("p64", _ksum([K.ExpSquaredKernel([v * (1 + 0.1 * i) for v in m8], ndim=8) for i in range(8)]), 8, 64),
        ("user_cauchy", 0.8 * K.CauchyKernel(metric=0.7, ndim=2), 2, 2),
    ]


@pytest.mark.parametrize("chunk", ["64", "192"])
@pytest.mark.parametrize("name,kernel,ndim,P", _param_kernels(), ids=[k[0] for k in _param_kernels()])
def test_streamed_parameter_counts(gpu, env, record_property, name, kernel, ndim, P, chunk):
    """1, 8, 9 and 64 parameters, and a user kernel, on approximate trees: g and diag against the HODLR's own K^-1
    (get_inverse, the unrestricted solve) contracted in longdouble, and against the resident path."""
    assert len(kernel.get_parameter_vector(include_frozen=True)) == P
    n = 300
    rng = np.random.default_rng(P + ndim)
    x = rng.uniform(0, 3, (n, ndim))
    x = x[np.argsort(x[:, 0])]
    yerr = 0.1 * np.ones(n)
    s = _solver(kernel, 40)
    s.compute(x, yerr)
    r = _rhs(x)
    which = np.ones(P, dtype=np.uint32)
    if P > 1:
        which[1] = 0
    alpha, g, diag = _streamed(s, r, which, env, chunk)
    assert np.all(g[which == 0] == 0.0)
    Kinv = s.get_inverse()
    errs = _grad_errors(kernel, x, Kinv, r, which, alpha, g, diag)
    a_res, g_res, d_res = _resident(s, r, which)
    A = np.outer(alpha, alpha) - Kinv
    dK = kernel.get_gradient(x, include_frozen=True)
    scale = np.einsum("ijk,ij->k", np.abs(dK), np.abs(A))
    scale[scale == 0] = 1
    errs["resident"] = float(np.max(np.abs(g - g_res) / scale))
    errs["diag_resident"] = _rel(diag, d_res)
    errs["alpha_equal"] = bool(np.array_equal(alpha, a_res))
    record_property("grad_err", errs["g"])
    record_property("diag_err", max(errs["diag"], errs["diag_resident"]))
    record_property("resident_err", errs["resident"])
    # (alpha is the resident path's, bit for bit; against K^-1 r it would measure the float64 solve's conditioning)
    assert errs["alpha_equal"], errs
    assert errs["g"] <= OWN_INV_TOL and errs["resident"] <= RESIDENT_TOL, errs
    assert errs["diag"] <= OWN_INV_TOL and errs["diag_resident"] <= OWN_INV_TOL, errs


# ---- 2. the restricted solve is the unrestricted one --------------------------------------------------------------

@pytest.mark.parametrize("rng_mode", ["pernode", "reference"])
@pytest.mark.parametrize("n,min_size", [(65, 16), (257, 32), (700, 50), (1024, 32)])
def test_restricted_solve_is_unrestricted(gpu, env, record_property, n, min_size, rng_mode):
    """No Gram half exceeds 512 rows, so the solve has no atomics and is deterministic: the streamed diagonal is
    alpha^2 - diag(get_inverse()) bit for bit, alpha is the resident path's, and g differs from the resident path's only
    by the summation order (every ordered pair vs each unordered pair once)."""
    from george_b200 import kernels as K
    kernel = 1.0 * K.ExpKernel(1.0) + 0.3 * K.Matern32Kernel(2.0)
    x, yerr = _exp_inputs(n, seed=3)
    s = _solver(kernel, min_size, rng_mode, tol=1e-10)
    s.compute(x, yerr)
    r = _rhs(x)
    which = np.ones(4, dtype=np.uint32)
    a_res, g_res, d_res = _resident(s, r, which)
    for chunk in ("64", "192"):
        alpha, g, diag = _streamed(s, r, which, env, chunk)
        assert np.array_equal(alpha, a_res)
        assert np.array_equal(diag, alpha ** 2 - np.diag(s.get_inverse()))
        A = np.outer(alpha, alpha) - s.get_inverse()
        scale = np.einsum("ijk,ij->k", np.abs(kernel.get_gradient(x, include_frozen=True)), np.abs(A))
        err = float(np.max(np.abs(g - g_res) / scale))
        record_property("resident_err", err)
        assert err <= RESIDENT_TOL, (g, g_res)


# ---- 3. chunk independence and determinism ------------------------------------------------------------------------

@pytest.mark.parametrize("n,min_size", [(300, 40), (1000, 60)])
def test_slab_width_independence(gpu, env, n, min_size):
    """g and diag are the same bits for every slab width (a multiple of 64) and for two identical calls; "100000" is
    one slab, the width the default rule picks at this n."""
    from george_b200 import kernels as K
    kernel = 1.0 * K.ExpKernel(1.0) + 0.3 * K.Matern32Kernel(2.0)
    x, yerr = _exp_inputs(n, seed=5)
    s = _solver(kernel, min_size, tol=1e-10)
    s.compute(x, yerr)
    r = _rhs(x)
    which = np.ones(4, dtype=np.uint32)
    ref = _streamed(s, r, which, env, "64")
    for chunk in ("64", "128", "448", "100000"):
        alpha, g, diag = _streamed(s, r, which, env, chunk)
        assert np.array_equal(alpha, ref[0]) and np.array_equal(g, ref[1]) and np.array_equal(diag, ref[2]), chunk


# ---- 4. GP level -------------------------------------------------------------------------------------------------

def test_gp_gradient_streamed(gpu, env, record_property):
    """GP.grad_log_likelihood with HODLRSolver, a fitted Model mean with a frozen parameter and a fitted non-constant
    white-noise model: streamed == resident up to the summation order, and both against longdouble."""
    import george_b200 as george
    from george_b200 import kernels
    from george_b200.modeling import Model

    class PolynomialModel(Model):
        parameter_names = ("m", "b")

        def get_value(self, t):
            return t.flatten() * self.m + self.b

    class LinearNoise(Model):
        parameter_names = ("c", "s")

        def get_value(self, t):
            return self.c + self.s * t.flatten()

    n = 700
    rng = np.random.default_rng(9)
    t = np.sort(rng.uniform(0, n / 50.0, n))
    y = 0.5 * t - 0.2 + np.sin(t) + 0.1 * rng.standard_normal(n)
    gp = george.GP(1.3 * kernels.ExpKernel(1.0), mean=PolynomialModel(m=0.4, b=0.1),
                   white_noise=LinearNoise(c=np.log(0.05), s=0.02), fit_white_noise=True,
                   solver=george.HODLRSolver, tol=1e-12, min_size=50, exhaust="dense")
    gp.freeze_parameter("mean:b")
    gp.compute(t, 0.05)
    resident = gp.grad_log_likelihood(y)
    assert gp.solver.solver.grad_timing()["slabs"] == 0
    env.setenv("BGP_GRAD_CHUNK", "128")
    streamed = gp.grad_log_likelihood(y)
    assert gp.solver.solver.grad_timing()["slabs"] == 6
    env.delenv("BGP_GRAD_CHUNK")

    # longdouble reference: K = k(t) + diag(yerr^2 + exp(wn)), parameters in (mean, white noise, kernel) order
    x = t[:, None]
    wn = gp._call_white_noise(x)
    Kd = gp.kernel.get_value(x)
    Kd[np.diag_indices(n)] += 0.05 ** 2 + np.exp(wn)
    L, d = hiprec.ldlt_ld(Kd)
    Kinv = hiprec.solve_ld(L * np.sqrt(d)[None, :], np.eye(n))
    alpha = Kinv @ (y - gp._call_mean(x)).astype(LD)
    A = np.outer(alpha, alpha) - Kinv
    dmu = gp._call_mean_gradient(x)
    dwn = gp._call_white_noise_gradient(x)
    mask = gp.kernel.unfrozen_mask
    dK = gp.kernel.get_gradient(x).astype(LD)
    ref = np.concatenate([dmu @ alpha, 0.5 * np.sum((np.exp(wn) * np.diag(A))[None, :] * dwn, axis=1),
                          0.5 * np.einsum("ijk,ij->k", dK, A)[mask]])
    scale = np.concatenate([np.abs(dmu) @ np.abs(alpha),
                            0.5 * np.sum(np.abs((np.exp(wn) * np.diag(A))[None, :] * dwn), axis=1),
                            0.5 * np.einsum("ijk,ij->k", np.abs(dK), np.abs(A))[mask]])
    assert len(ref) == len(gp) == len(streamed)
    err_ref = float(np.max(np.abs(streamed - ref) / scale))
    err_res = float(np.max(np.abs(streamed - resident) / scale))
    record_property("gp_err", err_ref)
    record_property("resident_err", err_res)
    assert err_ref <= GP_TOL and err_res <= RESIDENT_TOL, (streamed, resident, ref)


# ---- 5. full size, default selection -------------------------------------------------------------------------------

def test_full_size_default_selection(gpu, env, record_property):
    """N = 2^17 without BGP_GRAD_CHUNK: the resident K^-1 would be 128 GiB, so the default selection streams it.
    ConstantKernel * ExpKernel on sorted 1-D x is exactly rank 1 between halves, so the tree is exact at a tight tol.
    dK/dlogA = K - diag(sigma^2), so the amplitude entry of g obeys the identity
        g_logA = r.alpha - sum sigma_i^2 alpha_i^2 - N + sum sigma_i^2 (K^-1)_ii,  (K^-1)_ii = alpha_i^2 - diag_i
    with sigma^2 = yerr^2 + exp(white noise); the length-scale and white-noise entries of the GP gradient match centred
    differences of GP.log_likelihood."""
    import george_b200 as george
    from george_b200 import kernels
    n = 1 << 17
    rng = np.random.default_rng(17)
    t = np.sort(rng.uniform(0, n / 20.0, n))
    y = np.sin(0.3 * t) + 0.3 * rng.standard_normal(n)
    yerr = 0.1 * np.ones(n)
    kernel = kernels.ConstantKernel(log_constant=np.log(0.8)) * kernels.ExpKernel(1.5)
    gp = george.GP(kernel, white_noise=np.log(0.2 ** 2), fit_white_noise=True, solver=george.HODLRSolver,
                   tol=1e-12, min_size=256, exhaust="lowrank")
    gp.compute(t, yerr)
    native = gp.solver.solver
    assert max(nd["rank"] for nd in native.nodes() if not nd["is_leaf"]) <= 4

    which = np.ones(2, dtype=np.uint32)
    alpha, g, diag = gp.solver.grad_terms(y, which)
    timing = native.grad_timing()
    assert timing["slabs"] == n // 1024 and timing["slab_cols"] == 1024, timing
    sigma2 = yerr ** 2 + np.exp(gp.white_noise.get_parameter_vector()[0])
    kinv_diag = alpha ** 2 - diag
    terms = np.array([np.dot(y, alpha), -np.sum(sigma2 * alpha ** 2), -float(n), np.sum(sigma2 * kinv_diag)])
    err_id = abs(g[0] - np.sum(terms)) / np.sum(np.abs(terms))
    record_property("identity_err", float(err_id))
    assert err_id <= FULL_IDENTITY_TOL, (g[0], terms)

    grad = gp.grad_log_likelihood(y)  # (white noise, log constant, metric)
    # (not bit for bit: above 512 rows per Gram half the solve's Gram products add with atomics)
    assert abs(grad[1] - 0.5 * g[0]) <= 1e-12 * np.sum(np.abs(terms))
    p0 = gp.get_parameter_vector()
    h = 1e-4
    fd_err = 0.0
    for k in (0, 2):
        vals = []
        for sgn in (1, -1):
            p = p0.copy()
            p[k] += sgn * h
            gp.set_parameter_vector(p)
            vals.append(gp.log_likelihood(y))
        gp.set_parameter_vector(p0)
        fd = (vals[0] - vals[1]) / (2 * h)
        fd_err = max(fd_err, abs(grad[k] - fd) / max(1.0, abs(grad[k])))
    record_property("fd_err", fd_err)
    assert fd_err <= FULL_FD_TOL, (grad, fd_err)


# ---- 6. errors ----------------------------------------------------------------------------------------------------

def _raw_grad(native, n, P):
    from george_b200 import _lib
    which = np.ones(max(P, 1), dtype=np.uint32)
    r = np.ones(n)
    alpha, g, diag = np.zeros(n), np.zeros(max(P, 1)), np.zeros(n)
    st = native._lib.bgp_hodlr_grad_terms(native._ptr, _lib.ptr(which), _lib.ptr(r), _lib.ptr(alpha), _lib.ptr(g),
                                         _lib.ptr(diag))
    return st, _lib.last_error()


@pytest.mark.parametrize("chunk", [None, "64"])
def test_errors(gpu, env, chunk):
    """Uncomputed, sharded (before and after its top levels are finished) and P = 65: the same status and message with
    and without BGP_GRAD_CHUNK, and nothing launched before the P check."""
    import test_gpu_hodlr_shards as sh
    from george_b200 import _lib, kernels as K
    from george_b200.solvers._hodlr import HODLRSolver as Native
    lib = _lib.load()
    if chunk:
        env.setenv("BGP_GRAD_CHUNK", chunk)

    # (a new object may reuse a parked handle that still holds its last factorisation: release them)
    Native.release_parked()
    fresh = Native()
    assert _raw_grad(fresh, 8, 2) == (BGP_ERR_NOT_COMPUTED, "the solver has not been computed")

    kernel = 1.0 * K.ExpKernel(1.0)
    x, yerr = _exp_inputs(1024)
    Native.release_parked()
    pending = Native()
    _lib.check(sh._compute_status(pending, kernel, x, yerr, min_size=32, tol=1e-12, shard_rank=0, shard_count=2))
    assert _raw_grad(pending, 1024, 2) == (BGP_ERR_NOT_COMPUTED, "the solver has not been computed")
    shards = sh._shards(kernel, x, yerr, 2, min_size=32, tol=1e-12)
    for s in shards.handles:
        assert _raw_grad(s, 1024, 2) == (BGP_ERR_INVALID, "grad_terms is not available on a sharded factorisation")

    big = _ksum([K.Matern32Kernel([1.0] * 8, ndim=8) for _ in range(8)] + [K.ConstantKernel(log_constant=0.1, ndim=8)])
    assert len(big) == 65
    xb = np.random.default_rng(0).uniform(0, 1, (200, 8))
    Native.release_parked()
    native = Native()
    native.compute(big, xb, 0.1 * np.ones(200), min_size=50, tol=1e-12)
    before = lib.bgp_launch_count()
    assert _raw_grad(native, 200, 65) == (BGP_ERR_INVALID, "gradient supports at most 64 hyper-parameters")
    assert lib.bgp_launch_count() == before
