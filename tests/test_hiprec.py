# -*- coding: utf-8 -*-
"""The extended-precision reference of the factorisation tests (tests/hiprec.py) against LAPACK and against itself.
CPU only."""
import numpy as np
import pytest
import scipy.linalg

import hiprec


def _spd(n, seed):
    """Well-conditioned SPD matrix (cond <~ 10)."""
    rng = np.random.default_rng(seed)
    G = rng.normal(size=(n, n)) / np.sqrt(n)
    return G @ G.T + 2.0 * np.eye(n)


def test_longdouble_is_extended():
    assert np.finfo(np.longdouble).nmant >= 63
    assert np.finfo(np.longdouble).eps < 1.1e-19 * 1.01


@pytest.mark.parametrize("n", [1, 2, 65, 300])
def test_cholesky_against_lapack(n):
    K = _spd(n, n)
    L = hiprec.chol_ld(K)
    assert L.dtype == np.longdouble
    assert np.all(np.triu(L, 1) == 0)
    Lf = scipy.linalg.cholesky(K, lower=True)
    assert hiprec.rel_max(Lf, L) <= 1e-14
    assert abs(float(hiprec.logdet_ld(L)) - np.linalg.slogdet(K)[1]) <= 1e-13 * max(1.0, n)
    # L L^T reproduces K to extended precision: the reference is 1000x closer to exact than LAPACK
    LLt = L @ L.T
    assert float(np.max(np.abs(LLt - K.astype(np.longdouble)))) <= 1e-17 * np.max(np.abs(K))


@pytest.mark.parametrize("n", [1, 2, 65, 300])
def test_ldlt_against_cholesky(n):
    K = _spd(n, n + 1)
    L, d = hiprec.ldlt_ld(K)
    assert np.all(np.diag(L) == 1) and np.all(np.triu(L, 1) == 0)
    Lc = hiprec.chol_ld(K)
    assert hiprec.rel_max(L * np.sqrt(d)[None, :], Lc) <= 1e-17
    assert float(np.max(np.abs((L * d[None, :]) @ L.T - K.astype(np.longdouble)))) <= 1e-17 * np.max(np.abs(K))


@pytest.mark.parametrize("n,nrhs", [(1, 1), (65, 3), (300, 9)])
def test_residual_of_extended_solve(n, nrhs):
    K = _spd(n, 2 * n)
    B = np.random.default_rng(n).normal(size=(n, nrhs))
    X = hiprec.solve_ld(hiprec.chol_ld(K), B)
    assert hiprec.residual_ld(K, X, B) <= 1e-17
    # a float64 solve sits at float64 rounding, far above the extended one
    Xf = scipy.linalg.cho_solve(scipy.linalg.cho_factor(K, lower=True), B)
    assert hiprec.residual_ld(K, Xf, B) <= 1e-15


@pytest.mark.parametrize("n,nrhs,rows", [(1, 1, 512), (300, 9, 64), (300, 9, 300), (1031, 2, 512)])
def test_blocked_residual_matches_unblocked(n, nrhs, rows):
    """The row-blocked residual (for matrices whose longdouble copy does not fit) sums the same terms; both agree with a
    float64 evaluation to float64 rounding, and with each other to longdouble rounding."""
    K = _spd(n, 3 * n)
    rng = np.random.default_rng(n + rows)
    X = rng.normal(size=(n, nrhs))
    B = K @ X + 1e-8 * rng.normal(size=(n, nrhs))  # a residual far above float64 rounding
    full = hiprec.residual_ld(K, X, B)
    blocked = hiprec.residual_ld_blocked(K, X, B, rows=rows)
    assert abs(blocked - full) <= 1e-15 * full
    f64 = np.linalg.norm(K @ X - B) / (np.linalg.norm(K) * np.linalg.norm(X))
    assert abs(blocked - f64) <= 1e-3 * f64  # (the float64 product K @ X carries ~1e-14 of that residual's size)
    if n <= 300:  # an extended-precision solution: the residual is at longdouble rounding
        assert hiprec.residual_ld_blocked(K, hiprec.solve_ld(hiprec.chol_ld(K), B), B, rows=rows) <= 1e-17


def test_not_positive_definite_index():
    K = np.eye(5)
    K[1, 3] = K[3, 1] = 1.0
    K[3, 3] = 1.0
    with pytest.raises(np.linalg.LinAlgError, match="4-th leading minor"):
        hiprec.chol_ld(K)
