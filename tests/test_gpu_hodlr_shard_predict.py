# -*- coding: utf-8 -*-
"""GP.predict's variance and covariance on a sharded HODLR factorisation (``bgp_hodlr_predict_local_dev``, DESIGN.md
§5), on ONE device through the host-exchange protocol of ``test_gpu_hodlr_shards.py``.

With B = K(x, x*) and W = K^-1 B, shard s owns rows J_s and returns ``(prior ? K** : 0) - B[J_s]^T W[J_s]`` (COV) or
its diagonal (VAR).  The host solves B with the split solve (each shard keeps its own W, as P processes would), calls the
local entry on every shard with the prior on shard 0 only, and sums the parts in shard order.  The checks, for both
kinds:

* P = 1: on an unsharded handle the local entry, given apply_inverse's W, is ``bgp_hodlr_predict`` bit for bit;
* the sum over the sharded problems of ``test_gpu_hodlr_shards.CASES`` against a longdouble reference (exact-K trees),
  against each shard's own W contracted in longdouble, and against the unsharded handle;
* only the owned rows are read: NaN outside J_s in W leaves a shard's part unchanged, and ``solve_local_dev`` of a block
  that is NaN outside J_s gives the owned rows of the replicated block's solve;
* a ``kernel=`` other than the factorised one, repeatability, the error returns;
* ``GP.predict`` through a solver plug-in built on the shards, which never takes the host route;
* N = 2^17 on four shards.

Errors are measured on the prior's scale, ``max|out - ref| / max|K**|``, as in ``test_gpu_predict.py``.
"""

import ctypes as C

import numpy as np
import pytest

import hiprec
import test_gpu_hodlr_shard_grad as sg
import test_gpu_hodlr_shards as sh

pytestmark = pytest.mark.gpu

LD = np.longdouble

# bars: 10-100x the largest value measured on one H100 80GB HBM3 (SXM, 700 W power limit) over the cases of each test
LD_TOL = 5e-12         # sum of the parts vs the longdouble reference, exact-K trees           (measured 3.5e-13)
OWN_TOL = 5e-14        # a shard's part vs its own W contracted in longdouble                   (measured 1.9e-15)
SINGLE_TOL = 1e-10     # sum of the parts vs the unsharded bgp_hodlr_predict                    (measured 2.8e-12, cfg5)
OTHER_TOL = 5e-14      # the same with a kernel other than the factorised one                   (measured 1.5e-15)
GP_TOL = 5e-12         # GP.predict var / cov vs the unsharded GP and the longdouble reference  (measured 1.2e-13)
FULL_TOL = 1e-14       # N = 2^17, four shards, vs the unsharded bgp_hodlr_predict              (measured 2.8e-16)

KINDS = ["var", "cov"]
NS = 130               # test points of the sharded cases: two full 64-column groups and a ragged one
EXACT_MAX_N = 1024     # no atomics in the solve up to here: bit-exact comparisons
FILL = sh.FILL

BGP_ERR_INVALID, BGP_ERR_NOT_COMPUTED, BGP_ERR_DIM = 1, 3, 2


@pytest.fixture
def clean(monkeypatch):
    from george_b200.solvers._hodlr import HODLRSolver
    for var in ("BGP_PREDICT_CHUNK", "BGP_GRAD_CHUNK", "BGP_SMALL_RANK_LIMIT", "BGP_LEAF_COLS", "BGP_NO_GRAPH",
                "BGP_NO_CULL", "BGP_LEAF_FACTOR"):
        monkeypatch.delenv(var, raising=False)
    HODLRSolver.release_parked()
    yield monkeypatch
    HODLRSolver.release_parked()


def _lib():
    from george_b200 import _lib
    return _lib


def _xs(x, ns, seed):
    """ns test points over the range of x (one column sorted, so the test points cover every shard's rows)."""
    rng = np.random.default_rng(seed)
    lo, hi = x.min(axis=0) - 0.5, x.max(axis=0) + 0.5
    return rng.uniform(lo, hi, (ns, x.shape[1]))


def _B(kernel, x, xs):
    """K(x, x*) as the device builds it (kernel.get_value runs bgp_kmat_general)."""
    return kernel.get_value(xs, x).T


def _upload(W, nan_outside=None):
    """W (n x ns) into a column-major device block with ldw = n + PAD; the PAD rows hold FILL.  nan_outside=(row0,
    rows) replaces every row outside [row0, row0 + rows) with NaN."""
    n, ns = W.shape
    ldw = n + sh.PAD
    blk = np.full((ns, ldw), FILL)
    blk[:, :n] = W.T
    if nan_outside is not None:
        row0, rows = nan_outside
        blk[:, :row0] = np.nan
        blk[:, row0 + rows:] = np.nan
    d = sh._Dev(ns * ldw)
    d.upload(blk)
    return d, ldw


def _local(s, kernel, xs, what, W, add_prior, nan_outside=None):
    d, ldw = _upload(W, nan_outside)
    return s.predict_local(kernel, xs, what, d.p, ldw, add_prior)


def _predict(s, kernel, xs, what):
    """bgp_hodlr_predict on a native handle."""
    from george_b200.solvers.basic import BasicSolver
    return BasicSolver._predictive_call(s._lib.bgp_hodlr_predict, s._ptr, kernel, xs, what)


def _err(out, ref, kss):
    return float(np.max(np.abs(np.asarray(out, dtype=LD) - np.asarray(ref, dtype=LD))) / np.max(np.abs(kss)))


def _prior(kernel, xs, what):
    return kernel.get_value(xs, diag=True) if what == "var" else kernel.get_value(xs)


def _contract_ld(B, W, what):
    """B^T W (cov) or its diagonal (var) in longdouble."""
    B, W = np.asarray(B, dtype=LD), np.asarray(W, dtype=LD)
    return np.sum(B * W, axis=0) if what == "var" else B.T @ W


class _Parts(object):
    """The host side of one sharded prediction: W by the split solve (one copy per shard), the local entry on every
    shard with the prior on shard 0 only, and the parts summed in shard order."""

    def __init__(self, shards, kernel, xs, what, B, Ws=None):
        self.Ws = sh._sharded_solve(shards, B) if Ws is None else Ws
        self.parts = [_local(s, kernel, xs, what, W, k == 0) for k, (s, W) in enumerate(zip(shards.handles, self.Ws))]
        self.out = self.parts[0].copy()
        for p in self.parts[1:]:
            self.out += p


# ---- 1. P = 1 -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("chunk", [None, "64"])
@pytest.mark.parametrize("name,n,min_size,exhaust,tol", [
    ("exp", 1001, 60, "dense", 1e-12),
    ("m32", 1000, 64, "lowrank", 1e-10),
])
def test_unsharded_local_entry_is_predict(gpu, clean, name, n, min_size, exhaust, tol, chunk):
    """On an unsharded handle the own rows are [0, n): with add_prior = 1 and W = apply_inverse(K(x, x*)) the local
    entry returns bgp_hodlr_predict's bits (n <= 1024: the solve has no atomics, so its 64-column groups agree)."""
    kernel, x, yerr, _ = sh._problem(name, n)
    s = sh._single(kernel, x, yerr, min_size=min_size, tol=tol, exhaust=exhaust)
    if chunk is not None:
        clean.setenv("BGP_PREDICT_CHUNK", chunk)
    xs_all = _xs(x, 300, n)
    W_all = s.apply_inverse(_B(kernel, x, xs_all))
    for ns in (1, 63, 64, 65, 300):
        xs = xs_all[:ns]
        for what in KINDS:
            got = _local(s, kernel, xs, what, W_all[:, :ns], True)
            ref = _predict(s, kernel, xs, what)
            assert np.array_equal(got, ref), (ns, what)


# ---- 2 - 4. the sharded problems ------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", sh.CASES, ids=sh._case_id)
def test_sharded_prediction(gpu, clean, record_property, case):
    """The sum of the P shards' parts against the unsharded handle (every case), a longdouble reference (exact-K cases)
    and each shard's own W contracted in longdouble; a shard's part is unchanged by NaN outside its rows of W and by a
    second identical call; solve_local_dev reads only the owned rows."""
    name, n, min_size, P, exhaust, tol, small = case
    if small is not None:
        clean.setenv("BGP_SMALL_RANK_LIMIT", small)
    kernel, x, yerr, ref = sh._problem(name, n)
    opts = dict(min_size=min_size, tol=tol, exhaust=exhaust)
    single = sh._single(kernel, x, yerr, **opts)
    shards = sh._shards(kernel, x, yerr, P, **opts)
    xs = _xs(x, NS, n + P)
    B = _B(kernel, x, xs)
    kss = kernel.get_value(xs)
    Ws = sh._sharded_solve(shards, B)
    errs = {}
    for what in KINDS:
        parts = []
        for k, (s, W, (row0, rows)) in enumerate(zip(shards.handles, Ws, shards.ranges)):
            part = _local(s, kernel, xs, what, W, k == 0)
            J = slice(row0, row0 + rows)
            own = (_prior(kernel, xs, what).astype(LD) if k == 0 else 0) - _contract_ld(B[J], W[J], what)
            errs["own_" + what] = max(errs.get("own_" + what, 0.0), _err(part, own, kss))
            # only rows J of W are read, and a repeated call gives the same bits
            assert np.array_equal(_local(s, kernel, xs, what, W, k == 0, nan_outside=(row0, rows)), part), k
            assert np.array_equal(_local(s, kernel, xs, what, W, k == 0), part), k
            parts.append(part)
        out = parts[0].copy()
        for p in parts[1:]:
            out += p
        errs["single_" + what] = _err(out, _predict(single, kernel, xs, what), kss)
        if ref is not None:
            W_ld = hiprec.solve_ld(ref.Lc, B)
            full = _prior(kernel, xs, what).astype(LD) - _contract_ld(B, W_ld, what)
            errs["ld_" + what] = _err(out, full, kss)

    # solve_local_dev touches only the owned rows: a block that is NaN outside them solves to the same owned rows
    lib = _lib().load()
    ns = B.shape[1]
    for s, (row0, rows) in zip(shards.handles, shards.ranges):
        outs = []
        for nan in (False, True):
            blk = np.full((ns, n), np.nan) if nan else B.T.copy()
            blk[:, row0:row0 + rows] = B.T[:, row0:row0 + rows]
            d = sh._Dev(ns * n)
            d.upload(blk)
            _lib().check(lib.bgp_hodlr_solve_local_dev(s._ptr, d.p, ns, n))
            outs.append(d.download().reshape(ns, n)[:, row0:row0 + rows])
        assert np.all(np.isfinite(outs[1]))
        if n <= EXACT_MAX_N:
            assert np.array_equal(outs[0], outs[1])
        else:
            errs["local_solve_nan"] = max(errs.get("local_solve_nan", 0.0), sh._rel(outs[1], outs[0]))

    for k, v in errs.items():
        record_property(k, v)
    assert max(errs["own_var"], errs["own_cov"]) <= OWN_TOL, errs
    assert max(errs["single_var"], errs["single_cov"]) <= SINGLE_TOL, errs
    if ref is not None:
        assert max(errs["ld_var"], errs["ld_cov"]) <= LD_TOL, errs
    if "local_solve_nan" in errs:  # atomics in the solve above n = 1024 (measured 0)
        assert errs["local_solve_nan"] <= sh.SOLVE_TOL, errs


@pytest.mark.parametrize("P", [2, 4])
def test_other_kernel(gpu, clean, record_property, P):
    """GP.predict's `kernel=`: the test points and B use a kernel other than the factorised one."""
    from george_b200 import kernels as K
    kernel, x, yerr, _ = sh._problem("m32", 4097)
    opts = dict(min_size=64, tol=1e-10, exhaust="lowrank")
    other = 0.7 * K.Matern52Kernel(2.0) + 0.2 * K.ExpSquaredKernel(0.3)
    single = sh._single(kernel, x, yerr, **opts)
    shards = sh._shards(kernel, x, yerr, P, **opts)
    xs = _xs(x, NS, 5)
    B = _B(other, x, xs)
    kss = other.get_value(xs)
    Ws = sh._sharded_solve(shards, B)
    worst = 0.0
    for what in KINDS:
        got = _Parts(shards, other, xs, what, B, Ws)
        worst = max(worst, _err(got.out, _predict(single, other, xs, what), kss))
    record_property("other_kernel_err", worst)
    assert worst <= OTHER_TOL, worst


# ---- 5. errors ------------------------------------------------------------------------------------------------------

def test_local_entry_errors(gpu, clean):
    """NOT_COMPUTED on a fresh handle and on a shard waiting for its top levels; INVALID for an unknown kind, ns < 0,
    a null w_dev and ldw < N; DIM for a kernel of another dimension; each with nothing launched.  ns = 0 writes
    nothing.  A host-exchange shard's bgp_hodlr_predict keeps its status and message."""
    from george_b200 import kernels as K
    from george_b200._spec import flatten
    lib = _lib().load()
    n = 1024
    kernel, x, yerr, _ = sh._problem("exp", n)
    spec = flatten(kernel)
    xs = np.ascontiguousarray(_xs(x, 4, 0))
    out = np.full(16, -7.0)
    w = sh._Dev(4 * (n + 5))
    w.upload(np.ones(4 * (n + 5)))

    def call(h, ns=4, what=0, w_dev=w.p, ldw=n, sp=spec):
        return lib.bgp_hodlr_predict_local_dev(h._ptr, C.byref(sp), _lib().ptr(xs), ns, what, w_dev, ldw, 1,
                                               _lib().ptr(out))

    fresh = sh._native()
    assert call(fresh) == BGP_ERR_NOT_COMPUTED
    pending = sh._native()
    _lib().check(sh._compute_status(pending, kernel, x, yerr, min_size=32, tol=1e-12, shard_rank=1, shard_count=2))
    assert call(pending) == BGP_ERR_NOT_COMPUTED
    assert _lib().last_error() == "the solver has not been computed"

    shards = sh._shards(kernel, x, yerr, 2, min_size=32, tol=1e-12)
    spec2 = flatten(K.ExpKernel(1.0, ndim=2))
    for s in shards.handles + [sh._single(kernel, x, yerr, min_size=32, tol=1e-12)]:
        for kw, code in [(dict(what=2), BGP_ERR_INVALID), (dict(what=-1), BGP_ERR_INVALID),
                         (dict(ns=-1), BGP_ERR_INVALID), (dict(w_dev=None), BGP_ERR_INVALID),
                         (dict(ldw=n - 1), BGP_ERR_INVALID), (dict(sp=spec2), BGP_ERR_DIM)]:
            before = lib.bgp_launch_count()
            assert call(s, **kw) == code, kw
            assert lib.bgp_launch_count() == before, kw
        out[:] = -7.0
        before = lib.bgp_launch_count()
        assert call(s, ns=0, w_dev=None) == 0 and call(s, ns=0, what=1) == 0
        assert lib.bgp_launch_count() == before and np.all(out == -7.0)
        _lib().check(call(s, ldw=n + 5))  # ldw > N is accepted

    s = shards.handles[1]
    res = np.zeros(4)
    assert lib.bgp_hodlr_predict(s._ptr, C.byref(spec), _lib().ptr(xs), 4, 0, _lib().ptr(res)) == BGP_ERR_INVALID
    assert _lib().last_error() == "predict is not available on a sharded factorisation"


# ---- 6. GP level ----------------------------------------------------------------------------------------------------

class _PredictShards(sg._HostExchangeShards):
    """test_gpu_hodlr_shard_grad's host-exchange plug-in with ``predictive`` built on the local entry: the split solve
    of K(x, x*), every shard's part (the prior on shard 0), summed on the host."""

    def predictive(self, kernel, xs, what):
        xs = np.ascontiguousarray(xs, dtype=np.float64)
        xs = xs[:, None] if xs.ndim == 1 else xs
        x = self._x
        return _Parts(self.shards, kernel, xs, what, _B(kernel, x, xs)).out

    def compute(self, x, yerr):
        x = np.asarray(x, dtype=np.float64)
        self._x = x[:, None] if x.ndim == 1 else x
        super(_PredictShards, self).compute(x, yerr)


@pytest.mark.parametrize("P", [2, 4])
def test_gp_predict_on_shards(gpu, clean, record_property, P):
    """GP.predict(return_var=True) and (return_cov=True) on the shard plug-in against the unsharded GP and a longdouble
    reference; GP._predict_host is never called."""
    import george_b200 as george
    from george_b200 import kernels

    class Plugin(_PredictShards):
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

    gp = make(Plugin)
    single = make(george.HODLRSolver, rng_mode="pernode")

    def no_host(*args, **kwargs):
        raise AssertionError("GP.predict took the host route")

    clean.setattr(george.GP, "_predict_host", no_host)
    mu_v, var = gp.predict(y, ts, return_var=True)
    mu_c, cov = gp.predict(y, ts, return_cov=True)
    _, var1 = single.predict(y, ts, return_var=True)
    _, cov1 = single.predict(y, ts, return_cov=True)

    x = t[:, None]
    Kd = gp.kernel.get_value(x)
    Kd[np.diag_indices(n)] += gp._sigma(x) ** 2
    L = hiprec.chol_ld(Kd)
    xs = ts[:, None]
    B = _B(gp.kernel, x, xs)
    W = hiprec.solve_ld(L, B)
    kss = gp.kernel.get_value(xs)
    var_ref = _prior(gp.kernel, xs, "var").astype(LD) - _contract_ld(B, W, "var")
    cov_ref = kss.astype(LD) - _contract_ld(B, W, "cov")
    errs = {"var_ld": _err(var, var_ref, kss), "cov_ld": _err(cov, cov_ref, kss),
            "var_single": _err(var, var1, kss), "cov_single": _err(cov, cov1, kss)}
    for k, v in errs.items():
        record_property(k, v)
    assert np.array_equal(mu_v, mu_c)
    assert var.shape == (90,) and cov.shape == (90, 90)
    assert max(errs.values()) <= GP_TOL, errs


# ---- 7. larger size -------------------------------------------------------------------------------------------------

def test_four_shards_at_2_17(gpu, clean, record_property):
    """N = 2^17 on four shards at the default chunking: the sum of the parts agrees with the unsharded
    bgp_hodlr_predict for both kinds."""
    from george_b200 import kernels
    n, P, ns = 1 << 17, 4, 192
    rng = np.random.default_rng(17)
    x = np.sort(rng.uniform(0, n / 20.0, n))[:, None]
    yerr = 0.1 * np.ones(n)
    kernel = kernels.ConstantKernel(log_constant=np.log(0.8)) * kernels.ExpKernel(1.5)
    opts = dict(min_size=256, tol=1e-12, exhaust="lowrank")
    xs = _xs(x, ns, 3)
    kss = kernel.get_value(xs)
    single = sh._single(kernel, x, yerr, **opts)
    refs = {what: _predict(single, kernel, xs, what) for what in KINDS}
    del single
    shards = sh._shards(kernel, x, yerr, P, **opts)
    B = _B(kernel, x, xs)
    Ws = sh._sharded_solve(shards, B)
    errs = {}
    for what in KINDS:
        errs[what] = _err(_Parts(shards, kernel, xs, what, B, Ws).out, refs[what], kss)
    for k, v in errs.items():
        record_property(k, v)
    assert max(errs.values()) <= FULL_TOL, errs
