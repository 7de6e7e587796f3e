# -*- coding: utf-8 -*-
"""The dense and HODLR solvers on matrices of 2^31 entries and more, against the closed forms of ``ou_reference.py``.

From n = 46341 on, ``i * ld + j`` of an n x n matrix passes 2^31, so an index computed in 32 bits anywhere in the
kernel-matrix builds, the factorisation, the triangular solves, ``apply_sqrt``, the K^-1 formation or the gradient
contraction would show up here and nowhere else in the suite.  ``c * ExpKernel(m)`` on sorted 1-D points (gaps of
0.2 to 1.0 length scales, cond(K) <= 10) has an O(n) closed-form Cholesky factor, inverse, log-determinant, gradient
and prediction, so every check is against an exact answer in longdouble, whatever the size:

1. dense, n = 4161 (a small control, so that a failure only at the large size points at the size) and n = 46411
   (n^2 = 2.154e9, ragged against the 64-, 256- and 2048-column blocks): log det; columns of L through ``apply_sqrt``
   with one-hot rows on both sides of every block edge and past 2^31; ``apply_sqrt`` with random rows; ``apply_inverse``
   at 1, 4, 8, 9, 65 and 129 right-hand sides; ``dot_solve``; ``grad_terms`` (K^-1 of 2^31+ entries); the predictive
   mean and variance at 64 test points in several ``BGP_PREDICT_CHUNK`` chunks;
2. ``batch_log_likelihood`` with three members at n = 33000 in one chunk, so that the third member's matrix starts
   past 2^31 doubles: each member against the closed form, and bit for bit against the single path;
3. HODLR with ``exhaust="lowrank"`` (every node has rank 1, so the HODLR matrix is K to rounding): at N = 65536
   ``grad_terms`` with the resident K^-1 of 2^32 entries, against the closed form and against the streamed path; at
   N = 2^18 log det, solves at 1 and 65 right-hand sides, ``dot_solve``, the streamed ``grad_terms`` and the
   predictive mean and variance at 4096 test points.

Each test first reads the free device memory and skips, saying how much it found, when it is short of what the test
needs plus a margin.  Every error, the wall time and the device memory the test held are recorded with
``record_property``."""
import gc
import time

import numpy as np
import pytest

import ou_reference
from ou_reference import LD, OU

pytestmark = pytest.mark.gpu

# Bars, 10-30x the largest error measured on one H100 80GB HBM3 (SXM, 700 W power limit) over both dense sizes, the
# three batch members or both HODLR sizes:
DENSE_TOL = dict(
    logdet=1e-14,     # |logdet - ref| / |ref|                                                 (measured 3.2e-16)
    sqrt_col=2e-14,   # columns of L: max |out - L[:, j]| / max |L[:, j]|, worst column         (measured 1.0e-15)
    sqrt=3e-14,       # random rows: max |out - z L^T| / max |z L^T|                            (measured 1.4e-15)
    solve=3e-14,      # ||X - X_ref|| / ||X_ref||, worst right-hand side                       (measured 1.5e-15)
    dot=5e-15,        # |y^T K^-1 y - ref| / |ref|                                              (measured 1.1e-16)
    alpha=3e-14,      # ||alpha - ref|| / ||ref||                                               (measured 1.4e-15)
    g=1e-15,          # |g_p - ref| / sum |dK_p| |alpha alpha^T - K^-1| (bounded above)         (measured 2.5e-17)
    diag=5e-14,       # ||diag - ref|| / ||ref||                                                (measured 3.7e-15)
    mean=5e-14,       # max |mean - ref| / max |ref|                                            (measured 2.6e-15)
    var=5e-14)        # max |var - ref| / c                                                     (measured 2.1e-15)
BATCH_TOL = dict(logdet=5e-15, quad=5e-15)  # as the dense logdet and dot                      (measured 1.4e-16, 9.6e-17)
SINGLE_QUAD_TOL = 1e-13  # batch quad vs dot_solve (the batch tests' bar)
# HODLR, the dense measures (exhaust="lowrank", every node of rank 1):
#   logdet 1.2e-15, solve 1.2e-15, dot 3.1e-16, alpha 1.1e-15, g 1.7e-17, diag 2.5e-15, mean 2.5e-15, var 9.4e-16
HODLR_TOL = dict(logdet=3e-14, solve=3e-14, dot=1e-14, alpha=3e-14, g=1e-15, diag=5e-14, mean=5e-14, var=3e-14)
STREAM_TOL = 5e-15       # streamed vs resident grad_terms: alpha, diag relative 2-norm, g / scale  (measured 0)

MARGIN = 4 << 30         # bytes of free device memory kept in hand beyond a test's own estimate
GB = 1e9
KNOBS = ("BGP_PREDICT_CHUNK", "BGP_BATCH_CHUNK", "BGP_GRAD_CHUNK", "BGP_DENSE_OB", "BGP_DENSE_MB",
         "BGP_SMALL_RANK_LIMIT", "BGP_LEAF_COLS", "BGP_NO_GRAPH", "BGP_NO_CULL", "BGP_LEAF_FACTOR", "BGP_KMAT_GENERIC")


def _release():
    """Free the device memory that outlives a solver: the parked HODLR handles, the batch workspace and the blocks the
    library's default memory pool keeps cached (it never gives them back by itself).  Each test then starts from the
    memory the device really has free, and its own use shows in ``cudaMemGetInfo``."""
    import ctypes
    import torch
    from george_b200.solvers import basic
    from george_b200.solvers._hodlr import HODLRSolver
    basic._batch_handle = None
    gc.collect()
    HODLRSolver.release_parked()
    torch.cuda.synchronize()
    cu = ctypes.CDLL("libcuda.so.1")
    dev, pool = ctypes.c_int(), ctypes.c_void_p()
    assert cu.cuDeviceGet(ctypes.byref(dev), torch.cuda.current_device()) == 0
    assert cu.cuDeviceGetDefaultMemPool(ctypes.byref(pool), dev) == 0
    assert cu.cuMemPoolTrimTo(pool, ctypes.c_size_t(0)) == 0


@pytest.fixture
def env(monkeypatch):
    for var in KNOBS:
        monkeypatch.delenv(var, raising=False)
    _release()
    yield monkeypatch
    _release()


class _Memory(object):
    """Free device memory at the start and at each checkpoint (``cudaMemGetInfo``): ``held`` is the most the test held
    at a checkpoint, which with grow-only workspaces is the high-water mark of its solvers.  A checkpoint with a name
    also times the stage since the previous one (device work and reference alike)."""

    def __init__(self, need):
        import torch
        self._info = torch.cuda.mem_get_info
        self.free0, total = self._info()
        if self.free0 < need + MARGIN:
            pytest.skip("needs {0:.1f} GB of device memory plus a {1:.1f} GB margin; {2:.1f} of {3:.1f} GB free"
                        .format(need / GB, MARGIN / GB, self.free0 / GB, total / GB))
        self.held = 0
        self.t0 = self.t1 = time.time()
        self.stages = {}

    def check(self, stage=None):
        self.held = max(self.held, self.free0 - self._info()[0])
        if stage is not None:
            t = time.time()
            self.stages[stage] = t - self.t1
            self.t1 = t
        return self.held


def _record(record_property, errs, bars, mem):
    record_property("wall_s", round(time.time() - mem.t0, 1))
    record_property("device_gb_held", round(mem.held / GB, 2))
    for k, v in mem.stages.items():
        record_property("s:" + k, round(v, 2))
    for k, v in errs.items():
        record_property(k, "{0:.3g}".format(v))
    bad = {k: (v, bars[k.split(":")[0]]) for k, v in errs.items() if not v <= bars[k.split(":")[0]]}
    assert not bad, bad


def _rel2(X, Ref, axis=None):
    """``||X - Ref|| / ||Ref||`` in longdouble (per column with ``axis=0``, the worst one returned)."""
    Ref = np.asarray(Ref, dtype=LD)
    num = np.sqrt(np.sum((np.asarray(X, dtype=LD).reshape(Ref.shape) - Ref) ** 2, axis=axis))
    return float(np.max(num / np.sqrt(np.sum(Ref ** 2, axis=axis))))


def _absmax(X, Ref):
    """``max |X - Ref|`` in longdouble."""
    Ref = np.asarray(Ref, dtype=LD)
    return float(np.max(np.abs(np.asarray(X, dtype=LD).reshape(Ref.shape) - Ref)))


def _relmax(X, Ref):
    return _absmax(X, Ref) / float(np.max(np.abs(np.asarray(Ref, dtype=LD))))


def _grad_reference(ou, r):
    """``(alpha, g, diag)`` in longdouble and the scale of g: ``sum |dK_p| |alpha alpha^T - K^-1|`` per parameter,
    bounded above by ``|r| . |alpha| + n`` (log c) and ``(|alpha|^T D |alpha| + sum |K^-1| D) / 2`` (log m)."""
    alpha, g, diag = ou.grad_terms(r)
    aa = np.abs(alpha)
    _, e = ou.inv_tridiag()
    scale = np.array([np.abs(np.asarray(r, dtype=LD)) @ aa + ou.n,
                      (aa @ ou.apply_d(aa) + 2 * np.sum(np.abs(e) * ou.c * ou.rho[1:] * ou.delta[1:])) / 2])
    return alpha, g, diag, scale


def _grad_errors(ref, alpha, g, diag):
    """alpha and diag as relative 2-norms, g per parameter over its scale."""
    a_ref, g_ref, d_ref, scale = ref
    return {"alpha": _rel2(alpha, a_ref), "g": float(np.max(np.abs(np.asarray(g, dtype=LD) - g_ref) / scale)),
            "diag": _rel2(diag, d_ref)}


def _kernel(c, m):
    from george_b200 import kernels
    return c * kernels.ExpKernel(m)


# ---- 1. dense ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [4161, 46411])
def test_dense_against_closed_form(gpu, env, record_property, n):
    from george_b200 import BasicSolver
    # the factor and K^-1 of grad_terms, n^2 doubles each, and a 1 GiB test-point chunk
    mem = _Memory(2 * 8 * n * n + (1 << 30))
    c, m = 1.3, 0.8
    ell = np.sqrt(m)
    x = ou_reference.exp_problem(n, ell, seed=n, x0=-0.25 * n * ell)
    ou = OU(x, c, m)
    kernel = _kernel(c, m)
    rng = np.random.default_rng(n + 1)
    errs = {}

    s = BasicSolver(kernel)
    s.compute(x[:, None], 0.0)
    mem.check("compute")
    ld_ref = ou.logdet()
    errs["logdet"] = float(abs(s.log_determinant - ld_ref) / abs(ld_ref))

    # columns of L: both sides of the 64-, 2048- and 256-column block edges, around n/2 (the columns whose entries sit
    # past 2^31 at the large size) and the last 70 (the ragged last blocks)
    cols = sorted({0, 63, 64, 255, 256, 2047, 2048, n // 2 - 1, n // 2, n // 2 + 1} | set(range(n - 70, n)))
    E = np.zeros((len(cols), n))
    E[np.arange(len(cols)), cols] = 1.0
    out = s.apply_sqrt(E)
    Lc = ou.chol_columns(cols)
    errs["sqrt_col"] = max(_relmax(out[k], Lc[:, k]) for k in range(len(cols)))
    Z = rng.standard_normal((3, n))
    errs["sqrt"] = _relmax(s.apply_sqrt(Z), ou.sqrt_rows(Z))
    del E, out, Lc
    mem.check("apply_sqrt")

    for k in (1, 4, 8, 9, 65, 129):
        B = rng.standard_normal(n) if k == 1 else rng.standard_normal((n, k))
        errs["solve:{0}".format(k)] = _rel2(s.apply_inverse(B), ou.solve(B), axis=0)
    y = rng.standard_normal(n)
    q_ref = y.astype(LD) @ ou.solve(y)
    errs["dot"] = float(abs(s.dot_solve(y) - q_ref) / abs(q_ref))
    mem.check("solves")

    # predictions as GP.predict makes them: mean K(x*, x) alpha matrix-free, variance from the factor in chunks of 24
    # test points (64 = 24 + 24 + 16)
    xs = np.sort(rng.uniform(x[0], x[-1], 64))
    env.setenv("BGP_PREDICT_CHUNK", "24")
    var = s.predictive(kernel, xs[:, None], "var")
    env.delenv("BGP_PREDICT_CHUNK")
    mean = kernel.matvec(xs[:, None], x[:, None], s.apply_inverse(y).reshape(n))
    mean_ref, var_ref = ou.predict(xs, ou.solve(y))
    errs["mean"] = _relmax(mean, mean_ref)
    errs["var"] = _absmax(var, var_ref) / c
    mem.check("predict")

    alpha, g, diag = s.grad_terms(y, np.ones(2, dtype=np.uint32))
    mem.check("grad_terms")
    errs.update(_grad_errors(_grad_reference(ou, y), alpha, g, diag))
    del s
    _record(record_property, errs, DENSE_TOL, mem)


# ---- 2. batched member offsets -------------------------------------------------------------------------------------

def test_batch_member_offsets_past_2_31(gpu, env, record_property):
    from george_b200 import BasicSolver
    from george_b200._spec import flatten
    n, members = 33000, [(1.0, 1.0), (2.0, 0.64), (0.7, 1.2)]
    nb = len(members)
    assert (nb - 1) * n * n > 2 ** 31 > n * n  # the last member starts past 2^31 doubles; inside a member, it does not
    mem = _Memory(8 * nb * n * n + (1 << 30))
    x = ou_reference.exp_problem(n, 1.0, seed=n, x0=-0.3 * n)
    kernel = _kernel(1.0, 1.0)
    params = np.log(np.array(members))
    rng = np.random.default_rng(7)
    r = rng.standard_normal((nb, n))
    sig = np.zeros((nb, n))
    env.setenv("BGP_BATCH_CHUNK", str(nb))
    ld, q, info = BasicSolver.batch_log_likelihood(flatten(kernel), params, x, sig, r)
    assert np.all(info == 0), info
    held = mem.check("batch")
    assert held >= 8 * nb * n * n, held  # all three matrices were resident together, in one chunk
    env.delenv("BGP_BATCH_CHUNK")
    _release()

    errs = {}
    for b, (c, m) in enumerate(members):
        ou = OU(x, c, m)
        ld_ref = ou.logdet()
        q_ref = r[b].astype(LD) @ ou.solve(r[b])
        errs["logdet:{0}".format(b)] = float(abs(ld[b] - ld_ref) / abs(ld_ref))
        errs["quad:{0}".format(b)] = float(abs(q[b] - q_ref) / abs(q_ref))
        kernel.set_parameter_vector(params[b], include_frozen=True)
        s = BasicSolver(kernel)
        s.compute(x[:, None], sig[b])
        assert s.log_determinant == ld[b], (b, s.log_determinant, ld[b])
        q1 = s.dot_solve(r[b])
        assert abs(q[b] - q1) <= SINGLE_QUAD_TOL * abs(q1), (b, q[b], q1)
        del s
    mem.check("single")
    _record(record_property, errs, BATCH_TOL, mem)


# ---- 3. HODLR ------------------------------------------------------------------------------------------------------

def _hodlr(c, m, n, seed):
    import george_b200 as george
    ell = np.sqrt(m)
    x = ou_reference.exp_problem(n, ell, seed=seed, x0=-0.3 * n * ell)
    kernel = _kernel(c, m)
    s = george.HODLRSolver(kernel, min_size=256, tol=1e-12, seed=42, rng_mode="pernode", exhaust="lowrank")
    s.compute(x[:, None], np.zeros(n))
    ranks = {nd["rank"] for nd in s.solver.nodes() if not nd["is_leaf"]}
    assert ranks == {1}, ranks
    return x, kernel, s, OU(x, c, m)


def test_hodlr_resident_inverse_past_2_31(gpu, env, record_property):
    n = 65536
    # the resident K^-1 (2^32 doubles) and a streamed slab of 8192 columns
    mem = _Memory(8 * n * n + 8 * n * 8192 + (1 << 30))
    x, kernel, s, ou = _hodlr(0.9, 1.1, n, seed=n)
    y = np.random.default_rng(3).standard_normal(n)
    which = np.ones(2, dtype=np.uint32)
    res = s.grad_terms(y, which)
    assert s.solver.grad_timing()["slabs"] == 0  # the resident path
    mem.check("compute+resident")
    ref = _grad_reference(ou, y)
    errs = _grad_errors(ref, *res)
    env.setenv("BGP_GRAD_CHUNK", "8192")
    st = s.grad_terms(y, which)
    assert s.solver.grad_timing()["slabs"] == n // 8192
    env.delenv("BGP_GRAD_CHUNK")
    mem.check("streamed")
    errs.update({k + ":streamed": v for k, v in _grad_errors(ref, *st).items()})
    errs["resident_vs_streamed"] = max(_rel2(st[0], res[0]), _rel2(st[2], res[2]),
                                       float(np.max(np.abs(st[1] - res[1]) / ref[3])))
    del s
    _record(record_property, errs, dict(HODLR_TOL, resident_vs_streamed=STREAM_TOL), mem)


def test_hodlr_full_size_against_closed_form(gpu, env, record_property):
    n = 1 << 18
    # the factors, a 1 GiB K^-1 slab, a 1 GiB test-point chunk and the solve workspaces (6.7 GB measured)
    mem = _Memory(8 << 30)
    c, m = 1.4, 0.6
    x, kernel, s, ou = _hodlr(c, m, n, seed=n)
    rng = np.random.default_rng(5)
    errs = {}
    ld_ref = ou.logdet()
    errs["logdet"] = float(abs(s.log_determinant - ld_ref) / abs(ld_ref))
    for k in (1, 65):
        B = rng.standard_normal(n) if k == 1 else rng.standard_normal((n, k))
        errs["solve:{0}".format(k)] = _rel2(s.apply_inverse(B), ou.solve(B), axis=0)
    y = rng.standard_normal(n)
    q_ref = y.astype(LD) @ ou.solve(y)
    errs["dot"] = float(abs(s.dot_solve(y) - q_ref) / abs(q_ref))
    mem.check("compute+solves")

    res = s.grad_terms(y, np.ones(2, dtype=np.uint32))
    assert s.solver.grad_timing()["slabs"] > 1  # streamed by default above n = 65536
    mem.check("grad_terms")
    errs.update(_grad_errors(_grad_reference(ou, y), *res))

    xs = np.sort(rng.uniform(x[0], x[-1], 4096))
    var = s.predictive(kernel, xs[:, None], "var")
    mean = kernel.matvec(xs[:, None], x[:, None], s.apply_inverse(y).reshape(n))
    mem.check("predict")
    mean_ref, var_ref = ou.predict(xs, ou.solve(y))
    errs["mean"] = _relmax(mean, mean_ref)
    errs["var"] = _absmax(var, var_ref) / c
    del s
    _record(record_property, errs, HODLR_TOL, mem)
