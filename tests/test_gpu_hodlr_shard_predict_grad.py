# -*- coding: utf-8 -*-
"""GP.grad_predict's variance gradient on a sharded HODLR factorisation (``bgp_hodlr_predict_grad_local_dev``,
DESIGN.md §5), on ONE device through the host-exchange protocol of ``test_gpu_hodlr_shards.py``.

With B = K(x, x*) and W = K^-1 B, shard s owns rows J_s and returns ``var_s`` (``bgp_hodlr_predict_local_dev``'s VAR
part) and ``dvar_s,i = (prior ? d k(t_i, t_i) / d t_i : 0) - 2 sum_{j in J_s} d1 k(t_i, x_j) W_ji``.  The host solves B
with the split solve (each shard keeps its own W, as P processes would), calls the local entry on every shard with the
prior on shard 0 only, and sums the parts in shard order.  The checks:

* P = 1: on an unsharded handle the local entry, given apply_inverse's W, is ``bgp_hodlr_predict_grad`` bit for bit;
* the sum over the sharded problems of ``test_gpu_hodlr_shards.CASES`` against a longdouble reference (exact-K trees,
  analytic d1 k), against each shard's own W contracted in longdouble, and against the unsharded handle; each shard's
  ``var`` part is its ``predict_local`` VAR part bit for bit;
* only the owned rows of W are read;
* the prior's gradient on exactly one shard, with a kernel whose prior variance depends on the input;
* a ``kernel=`` other than the factorised one, 2-D and 3-D inputs, repeatability, the error returns;
* ``GP.grad_predict`` through a solver plug-in built on the shards, which never takes the host route;
* N = 2^17 on four shards.

Errors are measured on the prior's scale, ``max|out - ref| / max|K**|``, as in ``test_gpu_hodlr_shard_predict.py``.
"""

import ctypes as C

import numpy as np
import pytest

import hiprec
import test_gpu_hodlr_shard_predict as sp
import test_gpu_hodlr_shards as sh

pytestmark = pytest.mark.gpu

LD = np.longdouble

# bars: 10-100x the largest value measured on one H100 80GB HBM3 (SXM, 700 W power limit) over the cases of each test
LD_TOL = 5e-11         # sum of the parts vs the longdouble reference, exact-K trees           (measured 3.7e-12)
OWN_TOL = 5e-14        # a shard's dvar vs its own W contracted in longdouble                   (measured 6.9e-16)
SINGLE_TOL = 1e-10     # sum of the parts vs the unsharded bgp_hodlr_predict_grad               (measured 9.8e-12, cfg5)
PRIOR_TOL = 1e-14      # the prior on one shard vs on none, less the prior's terms              (measured 1.4e-16)
OTHER_TOL = 5e-13      # another kernel, 1-3 input dimensions, vs the unsharded handle          (measured 1.5e-14, 2-D)
GP_TOL = 5e-11         # GP dvar vs the unsharded GP and the longdouble reference               (measured 3.6e-12)
FD_TOL = 1e-7          # GP dvar vs central differences of the plug-in's own var, h = 1e-5    (measured 2.1e-9)
FULL_TOL = 1e-14       # N = 2^17, four shards, vs the unsharded bgp_hodlr_predict_grad        (measured 2.8e-16)

NS = sp.NS
FD_H = 1e-5

BGP_ERR_INVALID, BGP_ERR_NOT_COMPUTED, BGP_ERR_DIM = 1, 3, 2

clean = sp.clean


def _lib():
    from george_b200 import _lib
    return _lib


def _local(s, kernel, xs, W, add_prior, nan_outside=None):
    """(var, dvar) of one shard from its own W, uploaded with ldw = N + PAD."""
    d, ldw = sp._upload(W, nan_outside)
    return s.predict_grad_local(kernel, xs, d.p, ldw, add_prior)


def _predict_grad(s, kernel, xs):
    """bgp_hodlr_predict_grad on a native handle."""
    from george_b200.solvers.basic import BasicSolver
    return BasicSolver._predictive_grad_call(s._lib.bgp_hodlr_predict_grad, s._ptr, kernel, xs)


def _sum(parts):
    out = parts[0].copy()
    for p in parts[1:]:
        out += p
    return out


class _GradParts(object):
    """The host side of one sharded variance gradient: W by the split solve, the local entry on every shard with the
    prior on shard `prior_on` only (None: on no shard), the parts summed in shard order."""

    def __init__(self, shards, kernel, xs, B, Ws=None, prior_on=0):
        self.Ws = sh._sharded_solve(shards, B) if Ws is None else Ws
        self.parts = [_local(s, kernel, xs, W, k == prior_on) for k, (s, W) in enumerate(zip(shards.handles, self.Ws))]
        self.var = _sum([p[0] for p in self.parts])
        self.dvar = _sum([p[1] for p in self.parts])


def _dprior(kernel, xs):
    """d k(t, t) / d t (ns, ndim): the contraction's prior term alone, with no training points."""
    nd = xs.shape[1]
    return kernel.kernel.x1_gradient_matvec(xs, np.zeros((0, nd)), np.zeros(0), scale=0.0, add_prior=True)


def _exp_d1(c, xs, x):
    """d k(t_i, x_j) / d t_i of c * ExpKernel(1.0) in 1-D, in longdouble: (ns, n)."""
    d = xs[:, 0].astype(LD)[:, None] - x[:, 0].astype(LD)[None, :]
    return -c * np.exp(-np.abs(d)) * np.sign(d)


def _own_ld(kernel, xs, xJ, WJ, prior):
    """-2 sum_{j in J} d1 k(t_i, x_j) W_ji (+ the prior's gradient) in longdouble, from the device's d1 k in double
    (x1_gradient_general is the true derivative for the isotropic and axis-aligned metrics used here)."""
    G = kernel.kernel.x1_gradient_general(xs, xJ).astype(LD)   # (ns, nJ, nd)
    out = -2 * np.einsum("ijq,ji->iq", G, np.asarray(WJ, dtype=LD))
    return out + _dprior(kernel, xs).astype(LD) if prior else out


# ---- 1. P = 1 -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("chunk", [None, "64"])
@pytest.mark.parametrize("name,n,min_size,exhaust,tol", [
    ("exp", 1001, 60, "dense", 1e-12),
    ("m32", 1000, 64, "lowrank", 1e-10),
])
def test_unsharded_local_entry_is_predict_grad(gpu, clean, name, n, min_size, exhaust, tol, chunk):
    """On an unsharded handle the own rows are [0, n): with add_prior = 1, W = apply_inverse(K(x, x*)) and ldw > N the
    local entry returns bgp_hodlr_predict_grad's bits, var and dvar (n <= 1024: the solve has no atomics)."""
    kernel, x, yerr, _ = sh._problem(name, n)
    s = sh._single(kernel, x, yerr, min_size=min_size, tol=tol, exhaust=exhaust)
    if chunk is not None:
        clean.setenv("BGP_PREDICT_CHUNK", chunk)
    xs_all = sp._xs(x, 130, n)
    W_all = s.apply_inverse(sp._B(kernel, x, xs_all))
    for ns in (1, 63, 64, 65, 130):
        xs = xs_all[:ns]
        var, dvar = _local(s, kernel, xs, W_all[:, :ns], True)
        rvar, rdvar = _predict_grad(s, kernel, xs)
        assert np.array_equal(var, rvar), ns
        assert np.array_equal(dvar, rdvar), ns


# ---- 2 - 3. the sharded problems ------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", sh.CASES, ids=sh._case_id)
def test_sharded_gradient(gpu, clean, record_property, case):
    """The sum of the P shards' parts against the unsharded handle (every case), a longdouble reference (exact-K cases)
    and each shard's own W contracted in longdouble; a shard's var part is its predict_local VAR part, and its parts are
    unchanged by NaN outside its rows of W and by a second identical call."""
    name, n, min_size, P, exhaust, tol, small = case
    if small is not None:
        clean.setenv("BGP_SMALL_RANK_LIMIT", small)
    kernel, x, yerr, ref = sh._problem(name, n)
    opts = dict(min_size=min_size, tol=tol, exhaust=exhaust)
    single = sh._single(kernel, x, yerr, **opts)
    shards = sh._shards(kernel, x, yerr, P, **opts)
    xs = sp._xs(x, NS, n + P)
    B = sp._B(kernel, x, xs)
    kss = kernel.get_value(xs)
    Ws = sh._sharded_solve(shards, B)
    errs = {"own": 0.0}
    vparts, dparts = [], []
    for k, (s, W, (row0, rows)) in enumerate(zip(shards.handles, Ws, shards.ranges)):
        var, dvar = _local(s, kernel, xs, W, k == 0)
        assert var.shape == (NS,) and dvar.shape == (NS, x.shape[1])
        assert np.array_equal(var, sp._local(s, kernel, xs, "var", W, k == 0)), k
        J = slice(row0, row0 + rows)
        errs["own"] = max(errs["own"], sp._err(dvar, _own_ld(kernel, xs, x[J], W[J], k == 0), kss))
        # only rows J of W are read, and a repeated call gives the same bits
        for again in (_local(s, kernel, xs, W, k == 0, nan_outside=(row0, rows)), _local(s, kernel, xs, W, k == 0)):
            assert np.array_equal(again[0], var) and np.array_equal(again[1], dvar), k
        vparts.append(var)
        dparts.append(dvar)
    var, dvar = _sum(vparts), _sum(dparts)
    rvar, rdvar = _predict_grad(single, kernel, xs)
    errs["single_var"] = sp._err(var, rvar, kss)
    errs["single_dvar"] = sp._err(dvar, rdvar, kss)
    if ref is not None:  # 1.0 * ExpKernel(1.0): stationary, so the prior adds nothing to dvar
        W_ld = hiprec.solve_ld(ref.Lc, B)
        dvar_ld = -2 * np.einsum("ij,ji->i", _exp_d1(1.0, xs, x), W_ld)[:, None]
        errs["ld_dvar"] = sp._err(dvar, dvar_ld, kss)
    for k, v in errs.items():
        record_property(k, v)
    assert errs["own"] <= OWN_TOL, errs
    assert max(errs["single_var"], errs["single_dvar"]) <= SINGLE_TOL, errs
    if ref is not None:
        assert errs["ld_dvar"] <= LD_TOL, errs


# ---- 4. the prior on one shard --------------------------------------------------------------------------------------

@pytest.mark.parametrize("P", [2, 4])
def test_prior_on_exactly_one_shard(gpu, clean, record_property, P):
    """A kernel whose prior variance k(t, t) depends on t (a LocalGaussianKernel summed with a stationary one): with
    add_prior on any one shard the sum is the unsharded gradient; on none it differs from that by k(t, t) and its
    gradient, to rounding."""
    from george_b200 import kernels as K
    n = 1024
    x, yerr = sh.sw._inputs(n)
    kernel = 1.0 * K.ExpKernel(1.0) + 0.8 * K.LocalGaussianKernel(location=x[n // 3, 0], log_width=np.log(4.0))
    opts = dict(min_size=32, tol=1e-12, exhaust="dense")
    single = sh._single(kernel, x, yerr, **opts)
    shards = sh._shards(kernel, x, yerr, P, **opts)
    xs = sp._xs(x, NS, 7)
    B = sp._B(kernel, x, xs)
    kss = kernel.get_value(xs)
    Ws = sh._sharded_solve(shards, B)
    dprior = _dprior(kernel, xs)
    assert np.max(np.abs(dprior)) > 0.1  # the prior term is not trivially zero
    rvar, rdvar = _predict_grad(single, kernel, xs)
    none = _GradParts(shards, kernel, xs, B, Ws, prior_on=None)
    errs = {}
    for on in range(P):
        got = _GradParts(shards, kernel, xs, B, Ws, prior_on=on)
        errs["single_%d" % on] = max(sp._err(got.var, rvar, kss), sp._err(got.dvar, rdvar, kss))
        errs["none_%d" % on] = max(sp._err(got.var - none.var, kernel.get_value(xs, diag=True), kss),
                                   sp._err(got.dvar - none.dvar, dprior, kss))
    for k, v in errs.items():
        record_property(k, v)
    assert max(v for k, v in errs.items() if k.startswith("single")) <= SINGLE_TOL, errs
    assert max(v for k, v in errs.items() if k.startswith("none")) <= PRIOR_TOL, errs


# ---- 5. another kernel, 2-D and 3-D inputs --------------------------------------------------------------------------

def _problem_2d(n):
    from george_b200 import kernels as K
    rng = np.random.default_rng(n)
    x = rng.uniform(0, 4, (n, 2))
    x = x[np.argsort(x[:, 0])]
    return K.Matern52Kernel([0.5, 0.8], ndim=2), x, 0.1 * np.ones(n)


@pytest.mark.parametrize("ndim,P", [(1, 2), (1, 4), (2, 4), (3, 4)])
def test_other_kernel(gpu, clean, record_property, ndim, P):
    """GP.grad_predict's `kernel=`: the test points, B and the gradient use a kernel other than the factorised one; the
    same call twice gives the same bits."""
    from george_b200 import kernels as K
    if ndim == 1:
        kernel, x, yerr, _ = sh._problem("m32", 4097)
        opts = dict(min_size=64, tol=1e-10, exhaust="lowrank")
        other = 0.7 * K.Matern52Kernel(2.0) + 0.2 * K.ExpSquaredKernel(0.3)
    elif ndim == 2:
        kernel, x, yerr = _problem_2d(1500)
        opts = dict(min_size=75, tol=1e-8, exhaust="dense")
        other = 0.6 * K.ExpSquaredKernel([0.4, 0.9], ndim=2) + 0.3 * K.Matern32Kernel(1.5, ndim=2)
    else:
        kernel, x, yerr, _ = sh._problem("m52_3d", 1200)
        opts = dict(min_size=75, tol=1e-8, exhaust="dense")
        other = 0.9 * K.ExpSquaredKernel(0.6, ndim=3) + 0.1 * K.Matern32Kernel(0.3, ndim=3)
    single = sh._single(kernel, x, yerr, **opts)
    shards = sh._shards(kernel, x, yerr, P, **opts)
    xs = sp._xs(x, NS, 5)
    B = sp._B(other, x, xs)
    kss = other.get_value(xs)
    got = _GradParts(shards, other, xs, B)
    again = _GradParts(shards, other, xs, B, got.Ws)
    assert np.array_equal(got.var, again.var) and np.array_equal(got.dvar, again.dvar)
    rvar, rdvar = _predict_grad(single, other, xs)
    assert got.dvar.shape == (NS, ndim)
    err = max(sp._err(got.var, rvar, kss), sp._err(got.dvar, rdvar, kss))
    record_property("other_kernel_err", err)
    assert err <= OTHER_TOL, err


# ---- 6. errors ------------------------------------------------------------------------------------------------------

def test_local_entry_errors(gpu, clean):
    """NOT_COMPUTED on a fresh handle and on a shard waiting for its top levels; INVALID for ns < 0, a null w_dev,
    ldw < N and 9 input dimensions; DIM for a kernel of another dimension; each with nothing launched.  ns = 0 writes
    nothing.  A host-exchange shard's bgp_hodlr_predict_grad keeps its status and message."""
    from george_b200 import kernels as K
    from george_b200._spec import flatten
    lib = _lib().load()
    n = 1024
    kernel, x, yerr, _ = sh._problem("exp", n)
    spec = flatten(kernel)
    xs = np.ascontiguousarray(sp._xs(x, 4, 0))
    var, dvar = np.full(4, -7.0), np.full(4 * 9, -7.0)
    w = sh._Dev(4 * (n + 5))
    w.upload(np.ones(4 * (n + 5)))

    def call(h, ns=4, w_dev=w.p, ldw=n, sp_=spec, x_=xs):
        return lib.bgp_hodlr_predict_grad_local_dev(h._ptr, C.byref(sp_), _lib().ptr(x_), ns, w_dev, ldw, 1,
                                                    _lib().ptr(var), _lib().ptr(dvar))

    fresh = sh._native()
    assert call(fresh) == BGP_ERR_NOT_COMPUTED
    pending = sh._native()
    _lib().check(sh._compute_status(pending, kernel, x, yerr, min_size=32, tol=1e-12, shard_rank=1, shard_count=2))
    assert call(pending) == BGP_ERR_NOT_COMPUTED
    assert _lib().last_error() == "the solver has not been computed"

    shards = sh._shards(kernel, x, yerr, 2, min_size=32, tol=1e-12)
    spec2 = flatten(K.ExpKernel(1.0, ndim=2))
    for s in shards.handles + [sh._single(kernel, x, yerr, min_size=32, tol=1e-12)]:
        for kw, code in [(dict(ns=-1), BGP_ERR_INVALID), (dict(w_dev=None), BGP_ERR_INVALID),
                         (dict(ldw=n - 1), BGP_ERR_INVALID), (dict(sp_=spec2), BGP_ERR_DIM)]:
            before = lib.bgp_launch_count()
            assert call(s, **kw) == code, kw
            assert lib.bgp_launch_count() == before, kw
        var[:], dvar[:] = -7.0, -7.0
        before = lib.bgp_launch_count()
        assert call(s, ns=0, w_dev=None) == 0 and call(s, ns=0) == 0
        assert lib.bgp_launch_count() == before and np.all(var == -7.0) and np.all(dvar == -7.0)
        _lib().check(call(s, ldw=n + 5))  # ldw > N is accepted
        assert np.all(dvar[4:] == -7.0)   # (4, 1) written, nothing past it

    # 9 input dimensions: the handle factorises them, the gradient is refused before anything is launched
    rng = np.random.default_rng(9)
    k9 = K.ExpSquaredKernel(1.0, ndim=9, axes=[0, 4, 8])
    x9 = rng.uniform(size=(200, 9))
    x9 = x9[np.argsort(x9[:, 0])]
    s9 = sh._single(k9, x9, 0.1 * np.ones(200), min_size=32, tol=1e-12)
    xs9 = np.ascontiguousarray(rng.uniform(size=(4, 9)))
    before = lib.bgp_launch_count()
    assert call(s9, ldw=200, sp_=flatten(k9), x_=xs9) == BGP_ERR_INVALID
    assert lib.bgp_launch_count() == before
    assert "at most 8 dimensions" in _lib().last_error()

    s = shards.handles[1]
    assert lib.bgp_hodlr_predict_grad(s._ptr, C.byref(spec), _lib().ptr(xs), 4, _lib().ptr(var),
                                      _lib().ptr(dvar)) == BGP_ERR_INVALID
    assert _lib().last_error() == "predict_grad is not available on a sharded factorisation"


# ---- 7. GP level ----------------------------------------------------------------------------------------------------

class _PredictGradShards(sp._PredictShards):
    """test_gpu_hodlr_shard_predict's plug-in with ``predictive_grad`` built on the local entry.  ``apply_inverse`` of
    a matrix fails: GP.grad_predict's host route would solve K(x, x*) through it."""

    def predictive_grad(self, kernel, xs):
        xs = np.ascontiguousarray(xs, dtype=np.float64)
        xs = xs[:, None] if xs.ndim == 1 else xs
        got = _GradParts(self.shards, kernel, xs, sp._B(kernel, self._x, xs))
        return got.var, got.dvar

    def apply_inverse(self, y, in_place=False):
        if np.ndim(y) > 1:
            raise AssertionError("GP.grad_predict took the host route")
        return super(_PredictGradShards, self).apply_inverse(y, in_place)


@pytest.mark.parametrize("P", [2, 4])
def test_gp_grad_predict_on_shards(gpu, clean, record_property, P):
    """GP.grad_predict(return_var=True) on the shard plug-in: mu and var are the plug-in's GP.predict bit for bit, dvar
    agrees with the unsharded GP, a longdouble reference and central differences of the plug-in's own var."""
    import george_b200 as george
    from george_b200 import kernels

    class Plugin(_PredictGradShards):
        pass

    Plugin.P = P
    n = 700
    rng = np.random.default_rng(21)
    t = np.sort(rng.uniform(0, n / 50.0, n))
    y = np.sin(t) + 0.1 * rng.standard_normal(n)
    # test points half-way between training points at least 1e-3 apart: the Exp kernel's var has kinks at the x_j
    gaps = np.flatnonzero(np.diff(t) > 1e-3)
    ts = np.sort(0.5 * (t[gaps] + t[gaps + 1])[rng.choice(gaps.size, 90, replace=False)])

    def make(solver, **kw):
        gp = george.GP(1.3 * kernels.ExpKernel(1.0), solver=solver, tol=1e-12, min_size=50, exhaust="dense", **kw)
        gp.compute(t, 0.05)
        return gp

    gp = make(Plugin)
    single = make(george.HODLRSolver, rng_mode="pernode")
    mu, var, dmu, dvar = gp.grad_predict(y, ts, return_var=True)
    mu_p, var_p = gp.predict(y, ts, return_var=True)
    assert np.array_equal(mu, mu_p) and np.array_equal(var, var_p)
    assert dvar.shape == dmu.shape == (90, 1)
    _, _, _, dvar1 = single.grad_predict(y, ts, return_var=True)

    x = t[:, None]
    Kd = gp.kernel.get_value(x)
    Kd[np.diag_indices(n)] += gp._sigma(x) ** 2
    L = hiprec.chol_ld(Kd)
    xs = ts[:, None]
    W = hiprec.solve_ld(L, sp._B(gp.kernel, x, xs))
    dvar_ld = -2 * np.einsum("ij,ji->i", _exp_d1(1.3, xs, x), W)[:, None]
    kss = gp.kernel.get_value(xs)
    vp = gp.predict(y, ts + FD_H, return_var=True)[1]
    vm = gp.predict(y, ts - FD_H, return_var=True)[1]
    fd = (0.5 * (vp - vm) / FD_H)[:, None]
    errs = {"dvar_ld": sp._err(dvar, dvar_ld, kss), "dvar_single": sp._err(dvar, dvar1, kss),
            "dvar_fd": float(np.max(np.abs(dvar - fd)) / max(1.0, np.max(np.abs(fd))))}
    for k, v in errs.items():
        record_property(k, v)
    assert max(errs["dvar_ld"], errs["dvar_single"]) <= GP_TOL, errs
    assert errs["dvar_fd"] <= FD_TOL, errs


# ---- 8. larger size -------------------------------------------------------------------------------------------------

def test_four_shards_at_2_17(gpu, clean, record_property):
    """N = 2^17 on four shards at the default chunking: the sum of the parts agrees with the unsharded
    bgp_hodlr_predict_grad, var and dvar."""
    from george_b200 import kernels
    n, P, ns = 1 << 17, 4, 192
    rng = np.random.default_rng(17)
    x = np.sort(rng.uniform(0, n / 20.0, n))[:, None]
    yerr = 0.1 * np.ones(n)
    kernel = kernels.ConstantKernel(log_constant=np.log(0.8)) * kernels.ExpKernel(1.5)
    opts = dict(min_size=256, tol=1e-12, exhaust="lowrank")
    xs = sp._xs(x, ns, 3)
    kss = kernel.get_value(xs)
    single = sh._single(kernel, x, yerr, **opts)
    rvar, rdvar = _predict_grad(single, kernel, xs)
    del single
    shards = sh._shards(kernel, x, yerr, P, **opts)
    got = _GradParts(shards, kernel, xs, sp._B(kernel, x, xs))
    errs = {"var": sp._err(got.var, rvar, kss), "dvar": sp._err(got.dvar, rdvar, kss)}
    for k, v in errs.items():
        record_property(k, v)
    assert max(errs.values()) <= FULL_TOL, errs
