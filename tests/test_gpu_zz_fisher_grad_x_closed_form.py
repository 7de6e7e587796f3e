# -*- coding: utf-8 -*-
"""The Fisher information and the log-likelihood's input gradient against the closed forms of
``ou_reference.OU.fisher`` and ``OU.grad_x``, at the sizes where their device code runs paths that the small longdouble
tests of ``test_gpu_fisher.py``, ``test_gpu_batch_fisher.py`` and ``test_gpu_grad_x.py`` never reach.

``c * ExpKernel(m)`` on sorted 1-D points (gaps of 0.2 to 1.0 length scales, cond(K) <= 10) with ``yerr = 0`` and no
white noise has a tridiagonal K^-1, so the 3 x 3 F of (mean, log c, log m), every entry of ``dx`` and the gradient are
exact in O(n) longdouble at any size.  Every case runs through ``GP`` with a fitted constant mean (``r = y - mean`` a
sine plus seeded noise); ``grad`` from ``fisher_information(y)`` and ``grad_log_likelihood_x(y, return_gradient=True)``
is checked against ``OU.grad_terms`` as well.  Unlike the full-size tests' identities (the sum of F's scale block,
translation invariance of dx), which hold whatever the metric-derivative plane or a uniform scale of K^-1 or dx is,
these compare each entry with its true value.

1. dense ``fisher_information`` (``bgp_dense_fisher_terms``) at the split-K edges of its two n x n x n products
   (``predict_gemm_plan``, as ``test_gpu_zz_loo_closed_form.py``): the sizes must cover 1, 2, 3 and 4 slices on the
   device the test runs on.  Then n = 46345: n^2 passes 2^31 and the last 128-row tile has 9 rows; the factor, K^-1
   and the two product buffers hold 4 n^2 doubles (68.7 GB), against which the device memory held is checked (the
   call took 75 s on one H100 80GB HBM3, SXM, 700 W power limit);
2. ``batch_fisher_information`` with six members of different (c, m) at n = 2048 (2 slices) and 2049 (1 slice), each
   member against its own closed form;
3. dense ``grad_log_likelihood_x`` (``bgp_dense_grad_x_terms``: the resident ``alpha alpha^T - K^-1`` and the
   x-gradient matvec) at n = 129, 4161 and 46411 (past 2^31; the factor and K^-1, 2 n^2 doubles; 53 s there);
4. HODLR ``grad_log_likelihood_x`` (``exhaust="lowrank"``, every node of rank 1, so the HODLR matrix is K to rounding)
   on both sides of the resident/streamed switch, N = 65536 (resident K^-1, no slabs) and N = 65537 (streamed, 1984-column
   slabs), and N = 262181 = 2^18 + 37 in 2048-column slabs (129, the last of 37 columns, whose last 32-column tile has 5);
5. four host-exchange shards at N = 2^17 + 37, each contracting the input gradient of its own rows
   (``bgp_hodlr_grad_x_terms_local_dev``), the assembled dx against the closed form.

dx is compared entry by entry over ``OU.grad_x``'s scale (a bound of ``sum_j |A_ij| |dk_ij/dx_i|``), F entry by entry
relative to the entry.  Every error, the slice and slab counts, the wall time of each stage and the device memory held
are recorded with ``record_property``."""
import numpy as np
import pytest

from ou_reference import LD, OU
from test_gpu_zz_large_index import GB, _grad_reference, _Memory, _record
from test_gpu_zz_loo_closed_form import POOL_SLACK, SPLIT_SIZES, _gemm_slices, _problem, _sms, env  # noqa: F401

pytestmark = pytest.mark.gpu

# Bars, 10-30x the largest error measured on one H100 80GB HBM3 (SXM, 700 W power limit) over the sizes of a test:
# F each entry of (mean, log c, log m) relative to the entry; grad the GP's [mean, log c, log m] gradient (mean over
# sum |alpha|, the kernel entries as 2 grad against OU.grad_terms' g over its scale); dx per entry over OU.grad_x's scale.
TOL = dict(
    F=1e-14,      # (measured 4.6e-16; batch members 2.6e-16, past 2^31 1.6e-16)
    grad=1e-15,   # (measured 8.6e-17)
    dx=1e-13)     # (measured 6.9e-15; dense 4.0e-15, HODLR resident 4.6e-15, streamed 6.9e-15, shards 4.8e-15)
FD_SIZE = 46345          # dense Fisher past 2^31: 46345^2 = 2.148e9, 46345 = 362 * 128 + 9
GX_SIZE = 46411          # dense input gradient past 2^31, the LOO file's size
MEMBERS = [(1.3, 0.8), (0.6, 1.5), (2.2, 0.5), (1.0, 1.0), (0.9, 2.4), (1.7, 0.3)]


def _fisher_errors(F, grad, ou, r):
    """F's entries against ``OU.fisher`` (the mean-kernel entries must be exactly 0) and grad against
    ``OU.grad_terms``."""
    F = np.asarray(F)
    assert F.shape == (3, 3) and np.all(F[0, 1:] == 0) and np.all(F[1:, 0] == 0), F
    assert np.array_equal(F, F.T)
    ref = ou.fisher()
    err = max(float(abs(F[i, j] - ref[i, j]) / abs(ref[i, j])) for i, j in ((0, 0), (1, 1), (1, 2), (2, 2)))
    return {"F": err, "grad": _gp_grad_error(grad, ou, r)}


def _gp_grad_error(grad, ou, r):
    alpha, g, _, scale = _grad_reference(ou, r)
    return max(float(abs(grad[0] - np.sum(alpha)) / np.sum(np.abs(alpha))),
               float(np.max(np.abs(2 * np.asarray(grad[1:], dtype=LD) - g) / scale)))


def _dx_error(dx, ou, r):
    ref, scale = ou.grad_x(r)
    dx = np.asarray(dx)
    assert dx.shape == (ou.n, 1), dx.shape
    return float(np.max(np.abs(dx[:, 0].astype(LD) - ref) / scale))


def _label(errs, n):
    return {"{0}:{1}".format(k, n): v for k, v in errs.items()}


# ---- 1. dense Fisher -----------------------------------------------------------------------------------------------

def test_dense_fisher_split_k_edges(gpu, env, record_property):
    from george_b200 import BasicSolver
    sms = _sms()
    slices = {n: _gemm_slices(n, sms) for n in SPLIT_SIZES}
    record_property("sms", sms)
    record_property("slices", slices)
    assert {1, 2, 3, 4} <= set(slices.values()), slices
    mem = _Memory(1 << 30)
    c, m, mu = 1.3, 0.8, 0.4
    errs = {}
    for n in SPLIT_SIZES:
        gp, y, ou = _problem(n, c, m, mu, BasicSolver)
        grad, F = gp.fisher_information(y)
        errs.update(_label(_fisher_errors(F, grad, ou, y - mu), n))
        del gp
        mem.check(str(n))
    _record(record_property, errs, TOL, mem)


def test_dense_fisher_past_2_31(gpu, env, record_property):
    from george_b200 import BasicSolver
    n, P, nrow = FD_SIZE, 2, 2
    assert n * n > 2 ** 31 and n % 128 == 9
    # the factor, K^-1 and the product buffers P and T, n^2 doubles each: the products have one split-K slice
    mem = _Memory(4 * 8 * n * n)
    c, m, mu = 1.3, 0.8, 0.4
    gp, y, ou = _problem(n, c, m, mu, BasicSolver)
    mem.check("compute")
    assert _gemm_slices(n, _sms()) == 1
    grad, F = gp.fisher_information(y)
    held = mem.check("fisher")
    errs = _fisher_errors(F, grad, ou, y - mu)
    mem.check("reference")
    del gp
    # + the contraction's partials, the rows and their diagonals, alpha, the mean's solve and a few vectors
    workspace = 8 * (4 * n * n + (-(-n // 32)) ** 2 * P + nrow * (n + P) + 5 * n + 64)
    record_property("workspace_gb", round(workspace / GB, 2))
    assert held <= workspace + POOL_SLACK, (held, workspace)
    _record(record_property, errs, TOL, mem)


# ---- 2. batched Fisher ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n,nslices", [(2048, 2), (2049, 1)])
def test_batch_fisher_members(gpu, env, record_property, n, nslices):
    from george_b200 import BasicSolver
    assert _gemm_slices(n, _sms()) == nslices
    mem = _Memory(1 << 30)
    mu = 0.4
    gp, y, _ = _problem(n, 1.0, 1.0, mu, BasicSolver)
    assert gp.get_parameter_names() == ("mean:value", "kernel:k1:log_constant", "kernel:k2:metric:log_M_0_0")
    x = np.array(gp._x[:, 0])
    vectors = np.array([[mu, np.log(c), np.log(m)] for c, m in MEMBERS])
    p0 = gp.get_parameter_vector()
    grad, F = gp.batch_fisher_information(vectors, y)
    mem.check("batch")
    assert np.array_equal(gp.get_parameter_vector(), p0)
    errs = {}
    for b, (c, m) in enumerate(MEMBERS):
        errs.update(_label(_fisher_errors(F[b], grad[b], OU(x, c, m), y - mu), b))
    mem.check("reference")
    del gp
    _record(record_property, errs, TOL, mem)


# ---- 3. dense input gradient ---------------------------------------------------------------------------------------

def _grad_x_errors(gp, y, mu, ou):
    grad, dx = gp.grad_log_likelihood_x(y, return_gradient=True)
    r = y - mu
    return {"dx": _dx_error(dx, ou, r), "grad": _gp_grad_error(grad, ou, r)}


def test_dense_grad_x(gpu, env, record_property):
    from george_b200 import BasicSolver
    mem = _Memory(1 << 30)
    c, m, mu = 1.3, 0.8, 0.4
    errs = {}
    for n in (129, 4161):
        gp, y, ou = _problem(n, c, m, mu, BasicSolver)
        errs.update(_label(_grad_x_errors(gp, y, mu, ou), n))
        del gp
        mem.check(str(n))
    _record(record_property, errs, TOL, mem)


def test_dense_grad_x_past_2_31(gpu, env, record_property):
    from george_b200 import BasicSolver
    n, P = GX_SIZE, 2
    assert n * n > 2 ** 31
    # the factor and K^-1 (then alpha alpha^T - K^-1 in place), n^2 doubles each
    mem = _Memory(2 * 8 * n * n)
    c, m, mu = 1.3, 0.8, 0.4
    gp, y, ou = _problem(n, c, m, mu, BasicSolver)
    mem.check("compute")
    grad, dx = gp.grad_log_likelihood_x(y, return_gradient=True)
    held = mem.check("grad_x")
    errs = {"dx": _dx_error(dx, ou, y - mu), "grad": _gp_grad_error(grad, ou, y - mu)}
    mem.check("reference")
    del gp
    # + the contraction's partials, dx and a few vectors; the x-gradient matvec's row-split partials (a few n doubles)
    # are inside POOL_SLACK
    workspace = 8 * (2 * n * n + (-(-n // 32)) ** 2 * P + 6 * n + 64)
    record_property("workspace_gb", round(workspace / GB, 2))
    assert held <= workspace + POOL_SLACK, (held, workspace)
    _record(record_property, errs, TOL, mem)


# ---- 4. HODLR input gradient ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("n,chunk,slabs,last", [(65536, None, 0, None), (65537, None, 34, 65),
                                                 (262181, "2048", 129, 37)])
def test_hodlr_grad_x(gpu, env, record_property, n, chunk, slabs, last):
    import george_b200 as george
    # the resident K^-1 of 2^32 doubles at N = 65536; the factors, slabs and solve workspaces above
    mem = _Memory(8 * n * n + (1 << 30) if slabs == 0 else (8 << 30) if n > 100000 else (2 << 30))
    if chunk is not None:
        env.setenv("BGP_GRAD_CHUNK", chunk)
    if slabs:
        width = int(chunk) if chunk else max(64, (1 << 27) // n // 64 * 64)
        width = -(-width // 64) * 64
        assert (-(-n // width), n - (n - 1) // width * width) == (slabs, last), width
        record_property("slab_cols", width)
    c, m, mu = 1.4, 0.6, -0.3
    gp, y, ou = _problem(n, c, m, mu, george.HODLRSolver, min_size=256, tol=1e-12, seed=42, rng_mode="pernode",
                         exhaust="lowrank")
    ranks = {nd["rank"] for nd in gp.solver.solver.nodes() if not nd["is_leaf"]}
    assert ranks == {1}, ranks
    mem.check("compute")
    errs = _grad_x_errors(gp, y, mu, ou)
    timing = gp.solver.solver.grad_timing()
    record_property("slabs", timing["slabs"])
    assert timing["slabs"] == slabs, timing  # 0: the resident path
    mem.check("grad_x")
    del gp
    _record(record_property, errs, TOL, mem)


# ---- 5. host-exchange shards ---------------------------------------------------------------------------------------

def test_four_shards_grad_x(gpu, env, record_property):
    import test_gpu_hodlr_shards as sh
    from test_gpu_grad_x import SENTINEL, _dev_of
    import ou_reference
    from test_gpu_zz_large_index import _kernel
    n, P = (1 << 17) + 37, 4
    mem = _Memory(4 << 30)
    c, m, mu = 1.4, 0.6, -0.3
    ell = np.sqrt(m)
    x = ou_reference.exp_problem(n, ell, seed=n, x0=-0.3 * n * ell)
    y = mu + np.sin(x / ell) + 0.3 * np.random.default_rng(n + 1).standard_normal(n)
    r = y - mu
    ou = OU(x, c, m)
    shards = sh._shards(_kernel(c, m), x[:, None], np.zeros(n), P, min_size=256, tol=1e-12, exhaust="lowrank")
    mem.check("compute")
    alphas = [o[:, 0].copy() for o in sh._sharded_solve(shards, r[:, None])]
    which = np.ones(2, dtype=np.uint32)
    dx = np.full(n, np.nan)
    for s, (row0, rows), a in zip(shards.handles, shards.ranges, alphas):
        ad, dd = _dev_of(a, n), _dev_of(np.full(n, SENTINEL), n)
        s.grad_x_terms_local(ad.p, which, dd.p)
        d = dd.download()
        assert np.all(np.r_[d[:row0], d[row0 + rows:]] == SENTINEL)
        dx[row0:row0 + rows] = d[row0:row0 + rows]
    mem.check("grad_x")
    record_property("shard_rows", [rows for _, rows in shards.ranges])
    errs = {"dx": _dx_error(dx[:, None], ou, r)}
    del shards, alphas
    _record(record_property, errs, TOL, mem)
