# -*- coding: utf-8 -*-
"""Extended-precision references for the factorisation tests (test infrastructure; numpy only).

Everything here runs in ``np.longdouble``, which is the x87 80-bit format on x86-64 (64-bit mantissa, eps 1.1e-19):
three orders of magnitude below float64 rounding, so the distance of a float64 result from these references is the
float64 result's own error.  The factorisations are plain right-looking loops, O(n^3) in numpy's longdouble
arithmetic: ~1.4 s at n = 700, so use them for n <= ~800 and cache them per matrix.
"""
import numpy as np

LD = np.longdouble
assert np.finfo(LD).nmant >= 63, (
    "np.longdouble has a {0}-bit mantissa here: the extended-precision reference needs the 80-bit x87 format"
    .format(np.finfo(LD).nmant))


def chol_ld(K):
    """Lower Cholesky factor of the float64 matrix ``K`` (only its lower triangle is read), in longdouble."""
    A = np.tril(np.asarray(K, dtype=np.float64)).astype(LD)
    n = A.shape[0]
    for k in range(n):
        d = A[k, k]
        if not d > 0:
            raise np.linalg.LinAlgError("{0}-th leading minor is not positive definite".format(k + 1))
        lkk = np.sqrt(d)
        A[k, k] = lkk
        col = A[k + 1:, k] / lkk
        A[k + 1:, k] = col
        A[k + 1:, k + 1:] -= np.outer(col, col)  # the upper triangle is scratch
    return np.tril(A)


def ldlt_ld(K):
    """Un-pivoted ``K = L D L^T`` (L unit lower) of the float64 matrix ``K`` in longdouble; returns ``(L, d)``."""
    A = np.tril(np.asarray(K, dtype=np.float64)).astype(LD)
    n = A.shape[0]
    d = np.zeros(n, dtype=LD)
    for k in range(n):
        d[k] = A[k, k]
        col = A[k + 1:, k].copy()
        l = col / d[k]
        A[k + 1:, k] = l
        A[k + 1:, k + 1:] -= np.outer(l, col)
    L = np.tril(A, -1)
    L[np.diag_indices(n)] = 1
    return L, d


def logdet_ld(L):
    """``log det(L L^T)`` for a Cholesky factor, summed in longdouble."""
    return 2 * np.sum(np.log(np.diag(np.asarray(L)).astype(LD)))


def solve_ld(L, B):
    """``(L L^T)^-1 B`` by forward and backward substitution in longdouble (reference for the self-tests)."""
    L = np.asarray(L, dtype=LD)
    X = np.array(B, dtype=LD).reshape(L.shape[0], -1)
    n = L.shape[0]
    for i in range(n):
        X[i] = (X[i] - L[i, :i] @ X[:i]) / L[i, i]
    for i in range(n - 1, -1, -1):
        X[i] = (X[i] - L[i + 1:, i] @ X[i + 1:]) / L[i, i]
    return X.reshape(np.shape(B))


def residual_ld(K, X, B):
    """``||K X - B|| / (||K|| ||X||)`` (Frobenius norms) with the product and the sums accumulated in longdouble.
    A backward-stable float64 solve gives O(n eps) here whatever the condition number of K."""
    K = np.asarray(K, dtype=LD)
    X = np.asarray(X, dtype=LD).reshape(K.shape[0], -1)
    B = np.asarray(B, dtype=LD).reshape(K.shape[0], -1)
    R = K @ X - B
    nk = np.sqrt(np.sum(K * K))
    nx = np.sqrt(np.sum(X * X))
    return float(np.sqrt(np.sum(R * R)) / (nk * nx))


def residual_ld_blocked(K, X, B, rows=512):
    """``residual_ld`` with K converted to longdouble ``rows`` rows at a time: the same sums (to longdouble rounding)
    without a longdouble copy of the whole matrix (1 GB at n = 8194)."""
    K = np.asarray(K, dtype=np.float64)
    n = K.shape[0]
    X = np.asarray(X, dtype=LD).reshape(n, -1)
    B = np.asarray(B, dtype=LD).reshape(n, -1)
    r2 = LD(0)
    k2 = LD(0)
    for i0 in range(0, n, rows):
        Kb = K[i0:i0 + rows].astype(LD)
        R = Kb @ X - B[i0:i0 + rows]
        r2 += np.sum(R * R)
        k2 += np.sum(Kb * Kb)
    return float(np.sqrt(r2) / (np.sqrt(k2) * np.sqrt(np.sum(X * X))))


def rel_max(A, Ref):
    """``max|A - Ref| / max|Ref|``, evaluated in longdouble."""
    Ref = np.asarray(Ref, dtype=LD)
    return float(np.max(np.abs(np.asarray(A, dtype=LD) - Ref)) / np.max(np.abs(Ref)))
