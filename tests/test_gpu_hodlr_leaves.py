# -*- coding: utf-8 -*-
"""HODLR leaf factorisations and the leaf solve at their size switches, against an extended-precision reference.

Leaves of up to 768 rows are factorised by ``leaf_factor_dmma_kernel`` (csrc/hodlr_leaf.cuh), larger ones by
``leaf_build_factor_kernel`` (csrc/hodlr_kernels.cuh); ``BGP_LEAF_FACTOR=generic`` forces the latter at any size.  The
leaf solve stages column groups of 8 (32 with ``BGP_LEAF_COLS=32``) in shared memory, and 4, 2 or 1 for leaves above
3200 rows.  A tree whose root is a leaf (``min_size = N``) is exactly the un-pivoted LDL^T of K, so it is compared with
a longdouble LDL^T (n <= 800) or LAPACK at float64 rounding, not at the HODLR approximation bar.
"""
import numpy as np
import pytest
import scipy.linalg

import hiprec

pytestmark = pytest.mark.gpu

# bars: 10-60x the largest value measured on one H100 80GB HBM3 (SXM, 700 W power limit)
LOGDET_TOL = 2e-14      # |logdet - ref| / max(1, |ref|)                        (measured 5.5e-16)
SOLVE_TOL = 2e-12       # ||X - X_ref|| / ||X_ref||, cond(K) <~ 1e4              (measured 5.4e-14)
RESIDUAL_TOL = 3e-15    # ||K X - B|| / (||K|| ||X||), longdouble               (measured 6.0e-17)
TREE_LOGDET_TOL = 1e-13  # two-level trees (ACA at tol 1e-12): log-det vs oracle and dense  (measured 2.5e-15)
TREE_SOLVE_ORACLE_TOL = 5e-12  # ... solve vs the oracle                                 (measured 1.3e-13)
TREE_SOLVE_DENSE_TOL = 1e-9    # ... solve vs the dense one: the 1e-12 ACA truncation     (measured 2.8e-11)
WIDE_LOGDET_TOL = 1e-14  # BGP_LEAF_COLS=32 vs the default: log-det              (measured 1.6e-16)
WIDE_SOLVE_TOL = 1e-11   # ... and solves                                       (measured 1.7e-13)


def _kernel(kname):
    from george_b200 import kernels as K
    if kname == "m32_1d":
        return 1.0 * K.Matern32Kernel(1.0)
    if kname == "m52_3d":
        return 1.0 * K.Matern52Kernel(0.5, ndim=3)
    import conftest
    return dict(conftest.make_kernels())["sum_expsq_expsine2"]


def _inputs(kname, n, seed=0):
    rng = np.random.default_rng(seed + n)
    if kname == "m32_1d":
        x = np.sort(rng.uniform(0, max(1.0, n / 10.0), n))[:, None]
        yerr = 0.1 * np.ones(n)
    else:
        x = rng.uniform(0, max(1.0, (n / 4.0) ** (1.0 / 3.0)), (n, 3))
        x = x[np.argsort(x[:, 0])]
        yerr = 0.5 * np.ones(n)
    return x, yerr


_CACHE = {}


def _problem(kname, n):
    """(kernel, x, yerr, K, Lc) with Lc a Cholesky factor of K: longdouble (n <= 800) or LAPACK."""
    key = (kname, n)
    if key not in _CACHE:
        kernel = _kernel(kname)
        x, yerr = _inputs(kname, n)
        K = kernel.get_value(x)
        K[np.diag_indices(n)] += yerr ** 2
        if n <= 800:
            L, d = hiprec.ldlt_ld(K)
            Lc = L * np.sqrt(d)[None, :]
        else:
            Lc = scipy.linalg.cholesky(K, lower=True)
        _CACHE[key] = (kernel, x, yerr, K, Lc)
    return _CACHE[key]


def _solve_ref(Lc, B):
    if Lc.dtype == np.longdouble:
        return hiprec.solve_ld(Lc, B)
    return scipy.linalg.cho_solve((Lc, True), B)


def _rel(X, Xr):
    Xr = np.asarray(Xr, dtype=np.longdouble)
    return float(np.sqrt(np.sum((np.asarray(X, dtype=np.longdouble) - Xr) ** 2) / np.sum(Xr ** 2)))


def _check_exact_solver(s, K, Lc, nrhs_list, seed, record_property=None):
    """s factorises K exactly (one leaf, or a tree checked only through its residual elsewhere)."""
    n = K.shape[0]
    ld_ref = float(hiprec.logdet_ld(Lc))
    ld_err = abs(s.log_determinant - ld_ref) / max(1.0, abs(ld_ref))
    rng = np.random.default_rng(seed)
    fwd, res = {}, {}
    for nrhs in nrhs_list:
        B = rng.normal(size=(n, nrhs))
        X = s.apply_inverse(B)
        fwd[nrhs] = _rel(X, _solve_ref(Lc, B))
        if n <= 800 or nrhs in (1, 9):  # (the longdouble product costs O(n^2 nrhs))
            res[nrhs] = hiprec.residual_ld(K, X, B)
    if record_property is not None:
        record_property("logdet_err", ld_err)
        record_property("solve_err", max(fwd.values()))
        record_property("residual_err", max(res.values()))
    assert ld_err <= LOGDET_TOL, ld_err
    assert max(fwd.values()) <= SOLVE_TOL, fwd
    assert max(res.values()) <= RESIDUAL_TOL, res
    return s.log_determinant, X


SINGLE_N = [1, 2, 31, 32, 33, 95, 96, 97, 511, 767, 768, 769, 1000, 1500, 3200, 3201, 4000]


@pytest.mark.parametrize("n", SINGLE_N)
@pytest.mark.parametrize("kname", ["m32_1d", "sum3d"])
def test_single_leaf_tree_is_exact_ldlt(gpu, monkeypatch, record_property, kname, n):
    """min_size = N: the root is the only leaf, no low-rank node exists.  Above 3200 rows the leaf solve takes 4-column
    groups (the default 8 do not fit the 200 KB of shared memory)."""
    from george_b200.solvers._hodlr import HODLRSolver
    monkeypatch.delenv("BGP_LEAF_FACTOR", raising=False)
    monkeypatch.delenv("BGP_LEAF_COLS", raising=False)
    kernel, x, yerr, K, Lc = _problem(kname, n)
    s = HODLRSolver()
    s.compute(kernel, x, yerr, min_size=n, tol=1e-12, seed=42)
    nodes = s.nodes()
    assert len(nodes) == 1 and nodes[0]["is_leaf"]
    _check_exact_solver(s, K, Lc, [1, 7, 8, 9, 17], n, record_property)
    y = np.random.default_rng(n + 1).normal(size=n)
    q_ref = float(np.dot(y.astype(np.longdouble), np.asarray(_solve_ref(Lc, y), dtype=np.longdouble)))
    assert abs(s.dot_solve(y) - q_ref) <= SOLVE_TOL * abs(q_ref)


def test_leaf_too_large_for_the_solve_is_rejected_at_compute(gpu):
    """A leaf above 25600 rows does not fit the leaf solve even one column at a time: compute() says so."""
    from george_b200 import kernels as K
    from george_b200.solvers._hodlr import HODLRSolver
    n = 25601
    x = np.linspace(0.0, 1000.0, n)[:, None]
    s = HODLRSolver()
    with pytest.raises(ValueError, match="leaf size 25601 too large"):
        s.compute(1.0 * K.Matern32Kernel(1.0), x, 0.1 * np.ones(n), min_size=n, tol=1e-12, seed=42)
    assert not s.computed


@pytest.mark.parametrize("m", [1, 31, 32, 33, 64, 100, 255, 511, 768])
def test_generic_and_tensor_leaf_factor_agree(gpu, monkeypatch, m):
    """BGP_LEAF_FACTOR=generic runs leaf_build_factor_kernel where the DMMA kernel would run: both LDL^T
    implementations against the reference and against each other."""
    from george_b200.solvers._hodlr import HODLRSolver
    monkeypatch.delenv("BGP_LEAF_COLS", raising=False)
    kernel, x, yerr, K, Lc = _problem("m32_1d", m)
    out = {}
    for mode in ("tensor", "generic"):
        if mode == "generic":
            monkeypatch.setenv("BGP_LEAF_FACTOR", "generic")
        else:
            monkeypatch.delenv("BGP_LEAF_FACTOR", raising=False)
        s = HODLRSolver()
        s.compute(kernel, x, yerr, min_size=m, tol=1e-12, seed=42)
        out[mode] = _check_exact_solver(s, K, Lc, [1, 9], 7 * m)
    ld_t, X_t = out["tensor"]
    ld_g, X_g = out["generic"]
    assert abs(ld_t - ld_g) <= LOGDET_TOL * max(1.0, abs(ld_t))
    assert _rel(X_t, X_g) <= SOLVE_TOL


@pytest.mark.parametrize("n,min_size,leaf", [(1536, 768, 768), (1537, 768, 769), (3000, 1000, 1500)])
@pytest.mark.parametrize("kname", ["m32_1d", "m52_3d"])
def test_two_level_tree_across_the_leaf_switch(gpu, oracle, monkeypatch, record_property, kname, n, min_size, leaf):
    """Leaves of 768 rows take the DMMA kernel; one leaf of 769 sends every leaf to leaf_build_factor_kernel."""
    from george_b200.solvers._hodlr import HODLRSolver
    from george_b200._spec import flatten
    monkeypatch.delenv("BGP_LEAF_FACTOR", raising=False)
    monkeypatch.delenv("BGP_LEAF_COLS", raising=False)
    kernel, x, yerr, K, Lc = _problem(kname, n)
    s = HODLRSolver()
    s.compute(kernel, x, yerr, min_size=min_size, tol=1e-12, seed=42, rng_mode="pernode")
    nodes = s.nodes()
    assert max(nd["size"] for nd in nodes if nd["is_leaf"]) == leaf
    o = oracle.HODLR(flatten(kernel), x, yerr, min_size=min_size, tol=1e-12, seed=42, rng_mode=0)
    ld_ref = float(hiprec.logdet_ld(Lc))
    ld_o = abs(s.log_determinant - o.log_determinant) / abs(ld_ref)
    ld_d = abs(s.log_determinant - ld_ref) / abs(ld_ref)
    y = np.random.default_rng(n).normal(size=(n, 3))
    X = s.apply_inverse(y)
    Xo = np.stack([o.apply_inverse(y[:, c]) for c in range(3)], axis=1)
    Xd = np.asarray(_solve_ref(Lc, y), dtype=np.float64)
    so, sd = _rel(X, Xo), _rel(X, Xd)
    for name, v in (("logdet_vs_oracle", ld_o), ("logdet_vs_dense", ld_d), ("solve_vs_oracle", so),
                    ("solve_vs_dense", sd)):
        record_property(name, v)
    assert ld_o <= TREE_LOGDET_TOL and ld_d <= TREE_LOGDET_TOL
    assert so <= TREE_SOLVE_ORACLE_TOL and sd <= TREE_SOLVE_DENSE_TOL


def test_wide_leaf_solve_matches_default(gpu, monkeypatch, record_property):
    """BGP_LEAF_COLS=32 (the up-sweep and solves with > 8 columns in 32-column groups) against the default 8-column
    groups.  Every column goes through the same operations in the same order in both instantiations — only the number
    of columns a CTA holds differs.  The results are still not bit-identical: the level sweeps' Gram products
    (gram_tn_kernel) add their row chunks with atomicAdd, so two factorisations differ in the last bits whatever the
    leaf solve does (measured on the H100: log-dets 2 ulp, solutions 1.7e-13 apart)."""
    from george_b200 import kernels as K
    from george_b200.solvers._hodlr import HODLRSolver
    monkeypatch.delenv("BGP_LEAF_FACTOR", raising=False)
    n = 20000
    rng = np.random.default_rng(5)
    x = np.sort(rng.uniform(0, 10 * n / 1000, n))[:, None]
    yerr = 0.1 * np.ones(n)
    kernel = 1.0 * K.ExpSquaredKernel(1.0)
    y = rng.normal(size=(n, 20))
    res = {}
    for cols in ("8", "32"):
        monkeypatch.setenv("BGP_LEAF_COLS", cols)
        s = HODLRSolver()
        s.compute(kernel, x, yerr, min_size=100, tol=1e-10, seed=42, rng_mode="pernode")
        res[cols] = (s.log_determinant, s.apply_inverse(y), s.apply_inverse(y[:, 0]))
    assert max(nd["rank"] for nd in s.nodes()) > 0
    ld_d = abs(res["8"][0] - res["32"][0]) / abs(res["8"][0])
    x_d = max(_rel(res["8"][1], res["32"][1]), _rel(res["8"][2], res["32"][2]))
    record_property("logdet_diff", ld_d)
    record_property("solve_diff", x_d)
    assert ld_d <= WIDE_LOGDET_TOL
    assert x_d <= WIDE_SOLVE_TOL
