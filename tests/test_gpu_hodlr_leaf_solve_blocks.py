# -*- coding: utf-8 -*-
"""The HODLR leaf solve at its 32-row block boundaries, against an extended-precision un-pivoted LDL^T.

``leaf_solve_kernel`` (csrc/hodlr_kernels.cuh) stages each diagonal block through a two-buffer shared-memory ring and
updates the rows below in batches, and forms the backward dots of all 32 columns of a block at once.  A tree whose root
is a leaf (``min_size >= N``) is exactly the un-pivoted LDL^T of K, so its solves are compared with a longdouble LDL^T
(n <= 800) or LAPACK.  One ExpSquared leaf is ill-conditioned on purpose.  Two factorisations on one handle must agree
bit for bit: the solve sums every output in a fixed order.
"""
import numpy as np
import pytest
import scipy.linalg

import hiprec

pytestmark = pytest.mark.gpu

# bars as in test_gpu_hodlr_leaves.py (well-conditioned Matern leaves, cond(K) <~ 1e4)
LOGDET_TOL = 2e-14
SOLVE_TOL = 2e-12
RESIDUAL_TOL = 3e-15
TREE_SOLVE_DENSE_TOL = 1e-9  # two-level trees: the ACA truncation at tol 1e-12
EPS = np.finfo(np.float64).eps

LEAF_N = [1, 31, 32, 33, 100, 128, 200, 255, 256, 257, 768, 1000]  # 1000: leaf_build_factor_kernel (above 768 rows)
NRHS = [1, 2, 3, 8, 9, 29, 33]


def _matern(n, seed=0):
    from george_b200 import kernels as K
    rng = np.random.default_rng(seed + n)
    x = np.sort(rng.uniform(0, max(1.0, n / 10.0), n))[:, None]
    return 1.0 * K.Matern32Kernel(1.0), x, 0.1 * np.ones(n)


def _expsq(n, seed=0):
    """Closely spaced points under a long length scale with a small white-noise term: cond(K) ~ 1e7 and poorly
    conditioned 32 x 32 diagonal blocks of L."""
    from george_b200 import kernels as K
    rng = np.random.default_rng(seed + n)
    x = np.sort(rng.uniform(0, 5.0, n))[:, None]
    return 1.0 * K.ExpSquaredKernel(1.0), x, 0.003 * np.ones(n)


_CACHE = {}


def _problem(kind, n):
    key = (kind, n)
    if key not in _CACHE:
        kernel, x, yerr = (_matern if kind == "matern" else _expsq)(n)
        K = kernel.get_value(x)
        K[np.diag_indices(n)] += yerr ** 2
        if n <= 800:
            L, d = hiprec.ldlt_ld(K)
            Lc = L * np.sqrt(d)[None, :]
            blk = max(np.linalg.cond(np.asarray(L[k:k + 32, k:k + 32], dtype=np.float64)) for k in range(0, n, 32))
        else:
            Lc = scipy.linalg.cholesky(K, lower=True)
            blk = None
        _CACHE[key] = (kernel, x, yerr, K, Lc, blk)
    return _CACHE[key]


def _solve_ref(Lc, B):
    if Lc.dtype == np.longdouble:
        return hiprec.solve_ld(Lc, B)
    return scipy.linalg.cho_solve((Lc, True), B)


def _rel(X, Xr):
    Xr = np.asarray(Xr, dtype=np.longdouble)
    return float(np.sqrt(np.sum((np.asarray(X, dtype=np.longdouble) - Xr) ** 2) / np.sum(Xr ** 2)))


def _single_leaf(kernel, x, yerr, n):
    from george_b200.solvers._hodlr import HODLRSolver
    s = HODLRSolver()
    s.compute(kernel, x, yerr, min_size=n, tol=1e-12, seed=42)
    nodes = s.nodes()
    assert len(nodes) == 1 and nodes[0]["is_leaf"]
    return s


@pytest.mark.parametrize("cols", ["8", "32"])
@pytest.mark.parametrize("n", LEAF_N)
def test_single_leaf_solve_every_width(gpu, monkeypatch, record_property, n, cols):
    """Every right-hand-side count from 1 to 33 through one leaf, in 8- and 32-column groups."""
    monkeypatch.delenv("BGP_LEAF_FACTOR", raising=False)
    monkeypatch.setenv("BGP_LEAF_COLS", cols)
    kernel, x, yerr, K, Lc, _ = _problem("matern", n)
    s = _single_leaf(kernel, x, yerr, n)
    ld_err = abs(s.log_determinant - float(hiprec.logdet_ld(Lc))) / max(1.0, abs(float(hiprec.logdet_ld(Lc))))
    assert ld_err <= LOGDET_TOL, ld_err
    rng = np.random.default_rng(3 * n)
    worst_fwd, worst_res = 0.0, 0.0
    for nrhs in NRHS:
        B = rng.normal(size=(n, nrhs))
        X = s.apply_inverse(B)
        worst_fwd = max(worst_fwd, _rel(X, _solve_ref(Lc, B)))
        if n <= 800 or nrhs in (1, 9):
            worst_res = max(worst_res, hiprec.residual_ld(K, X, B))
    record_property("solve_err", worst_fwd)
    record_property("residual_err", worst_res)
    assert worst_fwd <= SOLVE_TOL, worst_fwd
    assert worst_res <= RESIDUAL_TOL, worst_res


@pytest.mark.parametrize("generic", [False, True])
@pytest.mark.parametrize("n", [200, 256, 768])
def test_ill_conditioned_expsq_leaf(gpu, monkeypatch, record_property, n, generic):
    """An ExpSquared leaf with cond(K) ~ 1e7 and ill-conditioned diagonal blocks of L: forward error within the LDL^T
    solve's own n eps cond(K), and a small backward error.  The same under the CUDA-core factorisation
    (BGP_LEAF_FACTOR=generic)."""
    monkeypatch.delenv("BGP_LEAF_COLS", raising=False)
    if generic:
        monkeypatch.setenv("BGP_LEAF_FACTOR", "generic")
    else:
        monkeypatch.delenv("BGP_LEAF_FACTOR", raising=False)
    kernel, x, yerr, K, Lc, blk = _problem("expsq", n)
    condK = np.linalg.cond(K)
    assert condK > 1e6 and blk > 10.0, (condK, blk)
    s = _single_leaf(kernel, x, yerr, n)
    B = np.random.default_rng(n).normal(size=(n, 9))
    X = s.apply_inverse(B)
    fwd = _rel(X, _solve_ref(Lc, B))
    res = hiprec.residual_ld(K, X, B)
    record_property("cond_K", condK)
    record_property("cond_L11_max", blk)
    record_property("solve_err", fwd)
    record_property("residual_err", res)
    assert fwd <= 50.0 * n * EPS * condK, (fwd, condK)
    assert res <= 100.0 * EPS * blk, (res, blk)


@pytest.mark.parametrize("nrhs", [1, 8, 29])
@pytest.mark.parametrize("n,min_size", [(512, 256), (1000, 200), (1537, 768)])
def test_small_tree_solve(gpu, monkeypatch, record_property, n, min_size, nrhs):
    """Two- and three-level trees: the up-sweep's per-depth column counts and the solve's leaf steps."""
    from george_b200.solvers._hodlr import HODLRSolver
    monkeypatch.delenv("BGP_LEAF_FACTOR", raising=False)
    monkeypatch.delenv("BGP_LEAF_COLS", raising=False)
    kernel, x, yerr, K, Lc, _ = _problem("matern", n)
    s = HODLRSolver()
    s.compute(kernel, x, yerr, min_size=min_size, tol=1e-12, seed=42, rng_mode="pernode")
    assert sum(1 for nd in s.nodes() if not nd["is_leaf"]) >= 1
    B = np.random.default_rng(n + nrhs).normal(size=(n, nrhs))
    err = _rel(s.apply_inverse(B), _solve_ref(Lc, B))
    record_property("solve_vs_dense", err)
    assert err <= TREE_SOLVE_DENSE_TOL, err


@pytest.mark.parametrize("generic", [False, True])
@pytest.mark.parametrize("kind,n", [("matern", 256), ("expsq", 700), ("matern", 1000)])
def test_second_compute_on_one_handle_is_bit_identical(gpu, monkeypatch, kind, n, generic):
    """compute() twice on one handle reuses the leaf-factor buffer and gives the same bits.  (Single-leaf trees:
    the level sweeps' Gram products add with atomics, so trees with low-rank nodes differ in the last bits anyway.)"""
    from george_b200.solvers._hodlr import HODLRSolver
    monkeypatch.delenv("BGP_LEAF_COLS", raising=False)
    if generic:
        monkeypatch.setenv("BGP_LEAF_FACTOR", "generic")
    else:
        monkeypatch.delenv("BGP_LEAF_FACTOR", raising=False)
    kernel, x, yerr = (_matern if kind == "matern" else _expsq)(n)
    y = np.random.default_rng(n).normal(size=n)
    s = HODLRSolver()
    out = []
    for _ in range(2):
        s.compute(kernel, x, yerr, min_size=n, tol=1e-10, seed=42)
        out.append((s.log_determinant, s.dot_solve(y)))
    assert out[0][0] == out[1][0]
    assert out[0][1] == out[1][1]
