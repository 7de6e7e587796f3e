# -*- coding: utf-8 -*-
"""The dense Cholesky (csrc/dense.cu) at its block-size boundaries, against an extended-precision reference.

``dense_potrf`` switches code at three nested block sizes: 64-column panels (NB), a delayed rank-MB update (MB = 256)
and a rank-OB update on the tensor pipe (OB = 2048).  ``BGP_DENSE_OB`` / ``BGP_DENSE_MB`` shrink the outer blocks so
that every update level and every ragged tail runs at small n, where the factor can be compared entry by entry with
a longdouble factorisation of the same float64 matrix (tests/hiprec.py); at n around 2048 and 4096 the default
blocking is compared with LAPACK.  The matrix is the one the device factorises: ``kernel.get_value`` runs the same
kernel-matrix build as ``BasicSolver.compute`` and ``yerr^2`` is added with the same single rounding.  (The CPU oracle's
kernel values agree with the device's only to ~1e-13, which would mask factorisation errors at this level.)
"""
import re

import numpy as np
import pytest
import scipy.linalg

import hiprec

pytestmark = pytest.mark.gpu

# bars: 10-50x the largest value measured on one H100 80GB HBM3 (SXM, 700 W power limit)
FACTOR_TOL = 5e-13      # max|L - L_ref| / max|L_ref|; also apply_sqrt      (measured 1.6e-14; 4.2e-14)
LOGDET_TOL = 5e-14      # |logdet - ref| / max(1, |ref|)                      (measured 1.1e-15)
RESIDUAL_TOL = 1e-14    # ||K X - B|| / (||K|| ||X||), longdouble             (measured 4.4e-16)
DOT_TOL = 5e-13         # |y^T K^-1 y - ref| / |ref|, cond(K) <~ 1e4         (measured 1.3e-14)

SMALL_N = [1, 63, 64, 65, 127, 129, 255, 257, 449, 577, 700]
LARGE_N = [2047, 2048, 2049, 2111, 2303, 4095, 4161]
BLOCKINGS = [("64", None), ("128", "64"), ("256", "64"), ("256", "128"), (None, None)]


def _kernel(kname):
    from george_b200 import kernels as K
    if kname == "m32_1d":
        return 1.0 * K.Matern32Kernel(1.0)
    import conftest
    return dict(conftest.make_kernels())["sum_expsq_expsine2"]


def _inputs(kname, n):
    rng = np.random.default_rng(1000 + n)
    if kname == "m32_1d":
        x = np.sort(rng.uniform(0, max(1.0, n / 10.0), n))[:, None]
        yerr = 0.1 * np.ones(n)
    else:
        x = rng.uniform(0, max(1.0, (n / 4.0) ** (1.0 / 3.0)), (n, 3))
        yerr = 0.5 * np.ones(n)
    return x, yerr


_CACHE = {}


def _problem(kname, n):
    """(kernel, x, yerr, K, L_ref) with L_ref the longdouble factor (n <= 800) or LAPACK's (larger n)."""
    key = (kname, n)
    if key not in _CACHE:
        kernel = _kernel(kname)
        x, yerr = _inputs(kname, n)
        K = kernel.get_value(x)
        K[np.diag_indices(n)] += yerr ** 2
        L_ref = hiprec.chol_ld(K) if n <= 800 else scipy.linalg.cholesky(K, lower=True)
        _CACHE[key] = (kernel, x, yerr, K, L_ref)
    return _CACHE[key]


def _factor(solver):
    from george_b200 import _lib
    n = solver._n
    L = np.empty((n, n), dtype=np.float64, order="F")
    _lib.check(solver._handle.lib.bgp_dense_export_factor(solver._handle.ptr, _lib.ptr(L)))
    return L


def _set_blocking(monkeypatch, ob, mb):
    for name, v in (("BGP_DENSE_OB", ob), ("BGP_DENSE_MB", mb)):
        if v is None:
            monkeypatch.delenv(name, raising=False)
        else:
            monkeypatch.setenv(name, v)


def _check_factor(s, K, L_ref, record_property):
    L = _factor(s)
    assert np.all(np.triu(L, 1) == 0.0)
    assert np.all(np.diag(L) > 0.0)
    err = hiprec.rel_max(L, L_ref)
    ld_ref = float(hiprec.logdet_ld(L_ref))
    ld_err = abs(s.log_determinant - ld_ref) / max(1.0, abs(ld_ref))
    record_property("factor_err", err)
    record_property("logdet_err", ld_err)
    assert err <= FACTOR_TOL
    assert ld_err <= LOGDET_TOL


@pytest.mark.parametrize("ob,mb", BLOCKINGS, ids=["OB64", "OB128-MB64", "OB256-MB64", "OB256-MB128", "default"])
@pytest.mark.parametrize("n", SMALL_N)
@pytest.mark.parametrize("kname", ["m32_1d", "sum3d"])
def test_factor_small_blocks(gpu, monkeypatch, record_property, kname, n, ob, mb):
    import george_b200 as george
    kernel, x, yerr, K, L_ref = _problem(kname, n)
    _set_blocking(monkeypatch, ob, mb)
    s = george.BasicSolver(kernel)
    s.compute(x, yerr)
    _check_factor(s, K, L_ref, record_property)


@pytest.mark.parametrize("n", LARGE_N)
@pytest.mark.parametrize("kname", ["m32_1d", "sum3d"])
def test_factor_default_blocks_large(gpu, monkeypatch, record_property, kname, n):
    import george_b200 as george
    kernel, x, yerr, K, L_ref = _problem(kname, n)
    _set_blocking(monkeypatch, None, None)
    s = george.BasicSolver(kernel)
    s.compute(x, yerr)
    _check_factor(s, K, L_ref, record_property)


@pytest.mark.parametrize("n", SMALL_N + [2049, 4161])
@pytest.mark.parametrize("kname", ["m32_1d", "sum3d"])
def test_solves(gpu, monkeypatch, record_property, kname, n):
    """apply_inverse with 1..8 right-hand sides (trsv_{fwd,bwd}_step_kernel<1>, <4>, <8>), 9 and 64 (trsv_block +
    gemm_sub), get_inverse, in-place and 3-D right-hand sides, dot_solve and apply_sqrt, all on the same factor."""
    import george_b200 as george
    kernel, x, yerr, K, L_ref = _problem(kname, n)
    _set_blocking(monkeypatch, None, None)
    s = george.BasicSolver(kernel)
    s.compute(x, yerr)
    rng = np.random.default_rng(n)
    res = []

    def check(X, B):
        res.append(hiprec.residual_ld(K, X, B))

    nrhs_list = [1, 2, 3, 4, 5, 8, 9, 64] if n <= 800 else [1, 3, 8, 9]
    for nrhs in nrhs_list:
        B = rng.normal(size=(n, nrhs))
        X = s.apply_inverse(B)
        assert X.shape == (n, nrhs)
        check(X, B)
    b = rng.normal(size=n)
    xb = s.apply_inverse(b)
    assert xb.shape == (n,)
    check(xb, b)
    # in place on a Fortran array: the result lands in the caller's buffer
    B = np.asfortranarray(rng.normal(size=(n, 5)))
    B0 = B.copy()
    out = s.apply_inverse(B, in_place=True)
    assert out is B
    check(B, B0)
    B3 = rng.normal(size=(n, 2, 3))
    X3 = s.apply_inverse(B3)
    assert X3.shape == (n, 2, 3)
    check(X3.reshape(n, 6, order="F"), B3.reshape(n, 6, order="F"))
    if n <= 800:
        Kinv = s.get_inverse()
        check(Kinv, np.eye(n))
    # dot_solve against the longdouble quadratic form of the extended-precision solve
    y = rng.normal(size=n)
    if n <= 800:
        q_ref = float(np.dot(y.astype(np.longdouble), hiprec.solve_ld(L_ref, y)))
    else:
        q_ref = float(y @ scipy.linalg.cho_solve((L_ref, True), y))
    q_err = abs(s.dot_solve(y) - q_ref) / abs(q_ref)
    # apply_sqrt: r @ L^T
    r = rng.normal(size=(3, n))
    want = r.astype(np.longdouble) @ np.asarray(L_ref, dtype=np.longdouble).T
    sq_err = float(np.max(np.abs(s.apply_sqrt(r) - want)) / np.max(np.abs(want)))
    record_property("residual_err", max(res))
    record_property("dot_err", q_err)
    record_property("sqrt_err", sq_err)
    assert max(res) <= RESIDUAL_TOL, res
    assert q_err <= DOT_TOL
    assert sq_err <= FACTOR_TOL


# ---- non positive-definite: an exact zero pivot reached through every level ------------------------------------------
# Points 50 apart under ExpSquared(1): r^2 >= 2500 and exp(-1250) is exactly 0, so K is the identity.  Moving point k
# onto point j makes K[j, k] = K[k, j] = 1 and the k-th pivot 1 - 1 * 1 = 0 exactly.  j and k are placed so that the
# zero is produced inside potf2 (same panel), by the panel solve + rank-64 update, the rank-MB update (k = 256) and the
# rank-OB update (k >= 2048).
NPD_N = 2100


@pytest.mark.parametrize("j,k", [(0, 1), (0, 63), (0, 64), (1, 65), (0, 256), (100, 2048), (7, 2049), (2047, 2048)])
def test_not_positive_definite_minor_index(gpu, monkeypatch, j, k):
    import george_b200 as george
    from george_b200 import kernels as KK
    _set_blocking(monkeypatch, None, None)
    n = NPD_N
    kernel = 1.0 * KK.ExpSquaredKernel(1.0)
    x = 50.0 * np.arange(n, dtype=np.float64)
    x[k] = x[j]
    Kh = kernel.get_value(x[:, None])
    assert np.count_nonzero(Kh - np.eye(n)) == 2
    with pytest.raises(np.linalg.LinAlgError) as ref:
        scipy.linalg.cholesky(Kh, lower=True)
    s = george.BasicSolver(kernel)
    with pytest.raises(np.linalg.LinAlgError) as got:
        s.compute(x[:, None], np.zeros(n))
    assert not s.computed
    # scipy states LAPACK's info as "<i>-th leading minor ..." or, since 1.15, "... info = [<i>] ..."
    minor = int(re.search(r"\d+", str(ref.value)).group())
    assert minor == k + 1
    assert str(got.value).startswith("{0}-th leading minor".format(minor)), str(got.value)

    gp = george.GP(kernel, white_noise=-800.0)  # exp(-800) == 0: nothing is added to the diagonal
    gp.compute(50.0 * np.arange(n, dtype=np.float64), 0.0)
    gp._x = x[:, None].copy()
    gp.computed = False
    assert gp.log_likelihood(np.ones(n), quiet=True) == -np.inf

    # the handle that failed factorises the next matrix correctly
    kernel2, x2, yerr2, K2, L2 = _problem("m32_1d", 2049)
    s.kernel = kernel2
    s.compute(x2, yerr2)
    assert s.computed
    assert hiprec.rel_max(_factor(s), L2) <= FACTOR_TOL
    b = np.random.default_rng(k).normal(size=2049)
    assert hiprec.residual_ld(K2, s.apply_inverse(b), b) <= RESIDUAL_TOL
