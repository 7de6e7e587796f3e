# -*- coding: utf-8 -*-
"""The log-likelihood gradient on a sharded HODLR factorisation (``bgp_hodlr_grad_terms_local_dev``, DESIGN.md §5),
on ONE device through the host-exchange protocol of ``test_gpu_hodlr_shards.py``.

Each shard streams K^-1 E_J over the columns J of its own rows: the identity is placed in J only, the row-restricted
solve runs its own leaves and owned levels and then the top levels, and the slab is contracted over the window J.  The
host forms alpha = K^-1 r with the split solve, calls the local entry on every shard, sums the partial g in shard order
and assembles the diag slices.  The checks, over the sharded problems of ``test_gpu_hodlr_shards.CASES``:

* P = 1: on an unsharded handle the local entry is the streamed ``bgp_hodlr_grad_terms``, bit for bit;
* the sum of the partials against a longdouble K^-1 (exact-K trees), against each shard's own K^-1 (the identity solved
  with the protocol, contracted in longdouble), and against the unsharded handle on the same problem;
* the restricted solve on a shard is the protocol's solve, bit for bit, where the solve has no atomics (n <= 1024), and
  rows outside a shard's slice are never written;
* a shard's partial g and diag do not depend on the slab width, and two calls agree bit for bit;
* frozen parameters, 1 to 64 parameters, and the error returns;
* ``GP.grad_log_likelihood`` through a solver plug-in built on the shards (the fused route, no K^-1);
* N = 2^17 on four shards at the default slab width.
"""

import functools
import operator

import numpy as np
import pytest

import hiprec
import test_gpu_hodlr_grad_stream as gs
import test_gpu_hodlr_shards as sh

pytestmark = pytest.mark.gpu

LD = np.longdouble

# bars: 10-100x the largest value measured on one H100 80GB HBM3 (SXM, 700 W power limit) over the cases of each test
GRAD_TOL = gs.GRAD_TOL     # sum of partials, alpha, diag vs longdouble K^-1, exact K     (measured 4.2e-12, alpha)
OWN_INV_TOL = 1e-14        # a shard's partial g / scale vs its own K^-1 in longdouble      (measured 1.4e-16)
SINGLE_G_TOL = 5e-13       # g / sum |dK| |A| vs the unsharded handle                       (measured 4.9e-15)
SINGLE_TOL = 1e-10         # alpha and diag (relative 2-norm) vs the unsharded handle       (measured 1.6e-12, alpha)
PARAM_TOL = 1e-14          # g / scale and diag for the 1 - 64 parameter kernels            (measured 1.8e-16)
GP_TOL = 2e-14             # GP gradient vs longdouble and vs the unsharded GP, per entry  (measured 4.4e-16)
FULL_TOL = 1e-14           # N = 2^17: |g - g_single| / max(1, |g_single|), diag and alpha (measured 1.7e-16)

SENTINEL = -123.25  # every diag row a shard must not write
LD_MAX_N = 1100     # longdouble contraction of a shard's own K^-1 up to here
EXACT_MAX_N = 1024  # no atomics in the solve up to here: bit-exact comparisons

BGP_ERR_INVALID, BGP_ERR_NOT_COMPUTED = 1, 3


@pytest.fixture
def clean(monkeypatch):
    from george_b200.solvers._hodlr import HODLRSolver
    for var in ("BGP_GRAD_CHUNK", "BGP_SMALL_RANK_LIMIT", "BGP_LEAF_COLS", "BGP_NO_GRAPH", "BGP_NO_CULL",
                "BGP_LEAF_FACTOR", "BGP_PREDICT_CHUNK"):
        monkeypatch.delenv(var, raising=False)
    HODLRSolver.release_parked()
    yield monkeypatch
    HODLRSolver.release_parked()


def _lib():
    from george_b200 import _lib
    return _lib


def _nparams(kernel):
    return len(kernel.get_parameter_vector(include_frozen=True))


def _grad_terms(s, r, which):
    """``bgp_hodlr_grad_terms`` on a native handle: (alpha, g, diag)."""
    n = r.size
    alpha, g, diag = np.empty(n), np.zeros(max(which.size, 1)), np.empty(n)
    r = np.ascontiguousarray(r, dtype=np.float64)
    _lib().check(s._lib.bgp_hodlr_grad_terms(s._ptr, _lib().ptr(which), _lib().ptr(r), _lib().ptr(alpha),
                                             _lib().ptr(g), _lib().ptr(diag)))
    return alpha, g[:which.size], diag


def _local(s, alpha, which):
    """The local entry with alpha uploaded and a diag buffer full of SENTINEL: (g_part, diag buffer after the call)."""
    n = alpha.size
    a = sh._Dev(n)
    a.upload(alpha)
    d = sh._Dev(n)
    d.upload(np.full(n, SENTINEL))
    g = s.grad_terms_local(a.p, which, d.p)
    return g, d.download()


class _Grad(object):
    """The host side of one sharded gradient: alpha by the split solve (each shard keeps its own copy, as P processes
    would), the local entry on every shard, the partials summed in shard order and the diag slices assembled."""

    def __init__(self, shards, r, which):
        n = r.size
        self.alphas = [o[:, 0].copy() for o in sh._sharded_solve(shards, r[:, None])]
        self.parts, self.buffers = [], []
        self.diag = np.full(n, np.nan)
        for s, (row0, rows), a in zip(shards.handles, shards.ranges, self.alphas):
            g, d = _local(s, a, which)
            outside = np.r_[d[:row0], d[row0 + rows:]]
            assert np.all(outside == SENTINEL), "a shard wrote diag rows outside its slice"
            self.parts.append(g)
            self.buffers.append(d)
            self.diag[row0:row0 + rows] = d[row0:row0 + rows]
        self.g = functools.reduce(operator.add, self.parts)
        self.alpha = self.alphas[0]


def _scaled(g, g_ref, scale):
    scale = np.where(scale == 0, 1, scale)
    return float(np.max(np.abs(np.asarray(g, dtype=LD) - np.asarray(g_ref, dtype=LD)) / scale)) if len(g) else 0.0


_KINV = {}


def _kinv_ld(key, ref, n):
    """The longdouble K^-1 from test_gpu_hodlr_sweeps' reference factorisation."""
    if key not in _KINV:
        _KINV[key] = hiprec.solve_ld(ref.Lc, np.eye(n))
    return _KINV[key]


def _shard_slabs(row0, rows, c):
    return -(-(row0 + rows - row0 // 64 * 64) // c)


# ---- 1. P = 1 -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("chunk", ["64", "128", "192"])
@pytest.mark.parametrize("name,n,min_size,exhaust,tol", [
    ("exp", 1001, 60, "dense", 1e-12),
    ("m32", 1000, 64, "lowrank", 1e-10),
    ("cfg5", 1000, 100, "lowrank", 1e-10),
])
def test_unsharded_local_entry_is_streamed_grad_terms(gpu, clean, name, n, min_size, exhaust, tol, chunk):
    """On an unsharded handle the own rows are [0, n): the local entry, given grad_terms' alpha, returns its g and
    diag bit for bit, with the same slabs (n <= 1024: the solve has no atomics, so two solves of a slab agree)."""
    kernel, x, yerr, _ = sh._problem(name, n)
    s = sh._single(kernel, x, yerr, min_size=min_size, tol=tol, exhaust=exhaust)
    r = gs._rhs(x)
    which = np.ones(_nparams(kernel), dtype=np.uint32)
    clean.setenv("BGP_GRAD_CHUNK", chunk)
    alpha, g, diag = _grad_terms(s, r, which)
    t_full = s.grad_timing()
    g_loc, d_loc = _local(s, alpha, which)
    t_loc = s.grad_timing()
    c = min(int(chunk), -(-n // 64) * 64)
    assert (t_loc["slabs"], t_loc["slab_cols"]) == (t_full["slabs"], t_full["slab_cols"]) == (-(-n // c), c), \
        (t_loc, t_full)
    assert np.array_equal(g_loc, g), (g_loc, g)
    assert np.array_equal(d_loc, diag)


# ---- 2 - 6. the sharded problems ------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", sh.CASES, ids=sh._case_id)
def test_sharded_gradient(gpu, clean, record_property, case):
    """The sum of the P shards' partials and the assembled diag against the unsharded handle (every case), a longdouble
    K^-1 (exact-K cases) and each shard's own K^-1 (n <= 1100); the diag slices bit for bit against the protocol's
    solve of the identity and across slab widths and repeated calls (n <= 1024)."""
    name, n, min_size, P, exhaust, tol, small = case
    if small is not None:
        clean.setenv("BGP_SMALL_RANK_LIMIT", small)
    kernel, x, yerr, ref = sh._problem(name, n)
    opts = dict(min_size=min_size, tol=tol, exhaust=exhaust)
    single = sh._single(kernel, x, yerr, **opts)
    shards = sh._shards(kernel, x, yerr, P, **opts)
    r = gs._rhs(x)
    which = np.ones(_nparams(kernel), dtype=np.uint32)
    got = _Grad(shards, r, which)
    c = shards.handles[0].grad_timing()["slab_cols"]
    for s, (row0, rows) in zip(shards.handles, shards.ranges):
        assert s.grad_timing()["slabs"] == _shard_slabs(row0, rows, c)
    errs = {}

    # against the unsharded handle, relative to sum |dK| |A| with A from its own K^-1
    a1, g1, d1 = _grad_terms(single, r, which)
    A1 = np.outer(a1, a1) - single.get_inverse()
    dK = kernel.get_gradient(x, include_frozen=True)
    scale = np.einsum("ijk,ij->k", np.abs(dK), np.abs(A1))
    errs["single_g"] = _scaled(got.g, g1, scale)
    errs["single_diag"] = gs._rel(got.diag, d1)
    errs["single_alpha"] = gs._rel(got.alpha, a1)
    del A1

    # against longdouble K^-1 (the HODLR matrix is K)
    if ref is not None:
        Kinv = _kinv_ld((name, n), ref, n)
        ld = gs._grad_errors(kernel, x, Kinv, r, which, got.alpha, got.g, got.diag)
        errs.update(("ld_" + k, v) for k, v in ld.items())

    # against each shard's own K^-1: the identity solved with the protocol, contracted in longdouble
    if n <= LD_MAX_N:
        X = sh._sharded_solve(shards, np.eye(n))
        errs["own"] = 0.0
        for k, ((row0, rows), a) in enumerate(zip(shards.ranges, got.alphas)):
            J = slice(row0, row0 + rows)
            A = np.outer(a, a[J]).astype(LD) - X[k][:, J].astype(LD)
            dKJ = dK[:, J]
            g_ref = np.einsum("ijk,ij->k", dKJ.astype(LD), A)
            own_scale = np.einsum("ijk,ij->k", np.abs(dKJ).astype(LD), np.abs(A))
            errs["own"] = max(errs["own"], _scaled(got.parts[k], g_ref, own_scale))
            if n <= EXACT_MAX_N:  # the restricted solve on a shard is the protocol's solve
                assert np.array_equal(got.buffers[k][J], a[J] ** 2 - np.diag(X[k])[J]), k

    # the partials do not depend on the slab width, and a repeated call gives the same bits
    if n <= EXACT_MAX_N:
        for chunk in (None, "64", "192", "100000"):
            if chunk is None:
                clean.delenv("BGP_GRAD_CHUNK", raising=False)
            else:
                clean.setenv("BGP_GRAD_CHUNK", chunk)
            for s, a, g_k, d_k in zip(shards.handles, got.alphas, got.parts, got.buffers):
                g2, d2 = _local(s, a, which)
                assert np.array_equal(g2, g_k) and np.array_equal(d2, d_k), chunk
        clean.delenv("BGP_GRAD_CHUNK", raising=False)

    for k, v in errs.items():
        record_property(k, v)
    assert errs["single_g"] <= SINGLE_G_TOL and errs["single_diag"] <= SINGLE_TOL, errs
    assert errs["single_alpha"] <= SINGLE_TOL, errs
    if ref is not None:
        assert max(errs["ld_" + k] for k in ("alpha", "g", "diag")) <= GRAD_TOL, errs
    if "own" in errs:
        assert errs["own"] <= OWN_INV_TOL, errs


# ---- 7. parameters and errors ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("name,kernel,ndim,P", gs._param_kernels(), ids=[k[0] for k in gs._param_kernels()])
def test_sharded_parameter_counts(gpu, clean, record_property, name, kernel, ndim, P):
    """1, 8, 9 and 64 parameters and a user kernel on two and four shards, one parameter frozen: it is exactly 0 in
    every partial, and the sum matches the unsharded handle."""
    n = 300
    rng = np.random.default_rng(P + ndim)
    x = rng.uniform(0, 3, (n, ndim))
    x = x[np.argsort(x[:, 0])]
    yerr = 0.1 * np.ones(n)
    opts = dict(min_size=40, tol=1e-12)
    single = sh._single(kernel, x, yerr, **opts)
    r = gs._rhs(x)
    which = np.ones(P, dtype=np.uint32)
    if P > 1:
        which[1] = 0
    a1, g1, d1 = _grad_terms(single, r, which)
    A1 = np.outer(a1, a1) - single.get_inverse()
    scale = np.einsum("ijk,ij->k", np.abs(kernel.get_gradient(x, include_frozen=True)), np.abs(A1))
    worst = 0.0
    for shard_count in (2, 4):
        got = _Grad(sh._shards(kernel, x, yerr, shard_count, **opts), r, which)
        for part in got.parts:
            assert part.shape == (P,) and np.all(part[which == 0] == 0.0)
        worst = max(worst, _scaled(got.g, g1, scale), gs._rel(got.diag, d1))
    record_property("param_err", worst)
    assert worst <= PARAM_TOL, worst


def test_local_entry_errors(gpu, clean):
    """NOT_COMPUTED on a fresh handle and on a shard waiting for its top levels; INVALID for a null alpha and for 65
    parameters, with nothing launched; a host-exchange shard's grad_terms keeps its status and message."""
    from george_b200 import kernels as K
    lib = _lib().load()
    n = 1024
    kernel, x, yerr, _ = sh._problem("exp", n)
    which = np.ones(2, dtype=np.uint32)
    g = np.zeros(2)
    a = sh._Dev(n)
    a.upload(np.ones(n))
    fresh = sh._native()
    assert lib.bgp_hodlr_grad_terms_local_dev(fresh._ptr, _lib().ptr(which), a.p, _lib().ptr(g), None) == \
        BGP_ERR_NOT_COMPUTED
    pending = sh._native()
    _lib().check(sh._compute_status(pending, kernel, x, yerr, min_size=32, tol=1e-12, shard_rank=1, shard_count=2))
    assert lib.bgp_hodlr_grad_terms_local_dev(pending._ptr, _lib().ptr(which), a.p, _lib().ptr(g), None) == \
        BGP_ERR_NOT_COMPUTED
    assert _lib().last_error() == "the solver has not been computed"

    shards = sh._shards(kernel, x, yerr, 2, min_size=32, tol=1e-12)
    s = shards.handles[1]
    before = lib.bgp_launch_count()
    assert lib.bgp_hodlr_grad_terms_local_dev(s._ptr, _lib().ptr(which), None, _lib().ptr(g), None) == BGP_ERR_INVALID
    assert lib.bgp_launch_count() == before
    r = np.ones(n)
    alpha, diag = np.zeros(n), np.zeros(n)
    assert lib.bgp_hodlr_grad_terms(s._ptr, _lib().ptr(which), _lib().ptr(r), _lib().ptr(alpha), _lib().ptr(g),
                                    _lib().ptr(diag)) == BGP_ERR_INVALID
    assert _lib().last_error() == "grad_terms is not available on a sharded factorisation"

    big = gs._ksum([K.Matern32Kernel([1.0] * 8, ndim=8) for _ in range(8)] + [K.ConstantKernel(log_constant=0.1, ndim=8)])
    assert len(big) == 65
    xb = np.random.default_rng(0).uniform(0, 1, (200, 8))
    xb = xb[np.argsort(xb[:, 0])]
    big_shards = sh._shards(big, xb, 0.1 * np.ones(200), 2, min_size=50, tol=1e-12)
    w65 = np.ones(65, dtype=np.uint32)
    g65 = np.zeros(65)
    ab = sh._Dev(200)
    ab.upload(np.ones(200))
    for hs in big_shards.handles:
        before = lib.bgp_launch_count()
        assert lib.bgp_hodlr_grad_terms_local_dev(hs._ptr, _lib().ptr(w65), ab.p, _lib().ptr(g65), None) == \
            BGP_ERR_INVALID
        assert _lib().last_error() == "gradient supports at most 64 hyper-parameters"
        assert lib.bgp_launch_count() == before


# ---- 8. GP level ----------------------------------------------------------------------------------------------------

class _HostExchangeShards(object):
    """A solver plug-in on P host-exchange shards in one process: the split solve for apply_inverse / dot_solve, and
    grad_terms from the local entry with a host sum.  get_inverse fails, so GP.grad_log_likelihood must take the fused
    route."""

    P = 2

    def __init__(self, kernel, min_size=50, tol=1e-12, exhaust="dense"):
        self.kernel, self.opts = kernel, dict(min_size=min_size, tol=tol, exhaust=exhaust)
        self.computed = False
        self.log_determinant = None

    def compute(self, x, yerr):
        x = np.asarray(x, dtype=np.float64)
        x = x[:, None] if x.ndim == 1 else x
        self._n = x.shape[0]
        self.shards = sh._shards(self.kernel, x, np.broadcast_to(yerr, (self._n,)), self.P, **self.opts)
        self.log_determinant = self.shards.log_determinant
        self.computed = True

    def apply_inverse(self, y, in_place=False):
        y = np.asarray(y, dtype=np.float64)
        return sh._sharded_solve(self.shards, y.reshape(self._n, -1))[0].reshape(y.shape)

    def dot_solve(self, y):
        return float(np.dot(y, self.apply_inverse(y)))

    def grad_terms(self, r, which):
        got = _Grad(self.shards, np.ascontiguousarray(r, dtype=np.float64), np.asarray(which, dtype=np.uint32))
        return got.alpha, got.g, got.diag

    def get_inverse(self):
        raise AssertionError("the gradient formed K^-1 instead of calling grad_terms")


@pytest.mark.parametrize("P", [2, 4])
def test_gp_gradient_on_shards(gpu, clean, record_property, P):
    """GP.grad_log_likelihood with a fitted mean model (one parameter frozen) and a fitted non-constant white-noise
    model on the shard plug-in, against the unsharded GP and a longdouble reference."""
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

    class Plugin(_HostExchangeShards):
        pass

    Plugin.P = P
    n = 700
    rng = np.random.default_rng(9)
    t = np.sort(rng.uniform(0, n / 50.0, n))
    y = 0.5 * t - 0.2 + np.sin(t) + 0.1 * rng.standard_normal(n)

    def make(solver, **kw):
        gp = george.GP(1.3 * kernels.ExpKernel(1.0), mean=PolynomialModel(m=0.4, b=0.1),
                       white_noise=LinearNoise(c=np.log(0.05), s=0.02), fit_white_noise=True, solver=solver,
                       tol=1e-12, min_size=50, exhaust="dense", **kw)
        gp.freeze_parameter("mean:b")
        gp.compute(t, 0.05)
        return gp

    gp = make(Plugin)
    grad = gp.grad_log_likelihood(y)
    single = make(george.HODLRSolver, rng_mode="pernode").grad_log_likelihood(y)

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
    assert len(ref) == len(gp) == len(grad) == len(single)
    err_ref = float(np.max(np.abs(grad - ref) / scale))
    err_single = float(np.max(np.abs(grad - single) / scale))
    record_property("gp_err", err_ref)
    record_property("single_err", err_single)
    assert err_ref <= GP_TOL and err_single <= GP_TOL, (grad, single, ref)


# ---- 9. larger size -------------------------------------------------------------------------------------------------

def test_four_shards_at_2_17(gpu, clean, record_property):
    """N = 2^17 on four shards at the default slab width (1024 columns): every shard streams only its 32 slabs, and the
    sum of the partials agrees with the unsharded streamed gradient; the amplitude entry meets the exact identity of
    test_gpu_hodlr_grad_stream.py::test_full_size_default_selection."""
    from george_b200 import kernels
    n, P = 1 << 17, 4
    rng = np.random.default_rng(17)
    x = np.sort(rng.uniform(0, n / 20.0, n))[:, None]
    y = np.sin(0.3 * x[:, 0]) + 0.3 * rng.standard_normal(n)
    yerr = 0.1 * np.ones(n)
    kernel = kernels.ConstantKernel(log_constant=np.log(0.8)) * kernels.ExpKernel(1.5)
    opts = dict(min_size=256, tol=1e-12, exhaust="lowrank")
    which = np.ones(2, dtype=np.uint32)
    single = sh._single(kernel, x, yerr, **opts)
    a1, g1, d1 = _grad_terms(single, y, which)
    t1 = single.grad_timing()
    assert (t1["slabs"], t1["slab_cols"]) == (128, 1024), t1
    del single
    shards = sh._shards(kernel, x, yerr, P, **opts)
    got = _Grad(shards, y, which)
    for s in shards.handles:
        assert (s.grad_timing()["slabs"], s.grad_timing()["slab_cols"]) == (32, 1024)
    errs = {"g": float(np.max(np.abs(got.g - g1) / np.maximum(1.0, np.abs(g1)))),
            "diag": gs._rel(got.diag, d1), "alpha": gs._rel(got.alpha, a1)}
    kinv_diag = got.alpha ** 2 - got.diag
    terms = np.array([np.dot(y, got.alpha), -np.sum(yerr ** 2 * got.alpha ** 2), -float(n),
                      np.sum(yerr ** 2 * kinv_diag)])
    errs["identity"] = float(abs(got.g[0] - np.sum(terms)) / np.sum(np.abs(terms)))
    for k, v in errs.items():
        record_property(k, v)
    assert max(errs["g"], errs["diag"], errs["alpha"]) <= FULL_TOL, errs
    assert errs["identity"] <= gs.FULL_IDENTITY_TOL, errs
