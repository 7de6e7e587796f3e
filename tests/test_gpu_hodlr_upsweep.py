# -*- coding: utf-8 -*-
"""The up-sweep and solve kernels at their tiling boundaries, against an extended-precision factorisation of the dense K.

``ExpKernel`` on sorted 1-D inputs is exactly rank 1 between the two halves of every node (exp(-(x_i - x_j)) =
e^{-x_i} e^{x_j}), so the HODLR matrix equals K to rounding whichever way the ACA finishes:
* ``exhaust="dense"``: every node runs out of rows and stores its block exactly, rank = floor(size / 2); the level ranks
  are then set through N and min_size, which puts ``gram_tn_small_kernel`` (2r <= 16, instantiated for r <= 2, 4, 8) and
  ``gram_tn_kernel`` (2r > 16) on the levels of one tree, with r exactly at the switch among them;
* ``exhaust="lowrank"``: every node keeps rank 1 at any size, so nodes of thousands of rows that are not multiples of the
  1024-row tiles of ``finalize_panels_kernel`` and ``gram_tn_small_kernel`` go through the small-rank path.
The right-hand-side counts run every leaf-solve instantiation (1, 2, 4 and 8 columns) with one and several column
groups per leaf; the up-sweep itself solves the leaves against all ancestor columns.
"""

import numpy as np
import pytest
import scipy.linalg

import hiprec

pytestmark = pytest.mark.gpu

LD = np.longdouble

# the bars of test_gpu_hodlr_sweeps.py (same problem family, same kernels)
LOGDET_TOL = 2e-13      # |logdet - ref| / max(1, |ref|)
SOLVE_TOL = 1e-11       # ||X - X_ref|| / ||X_ref||; also dot_solve
RESIDUAL_TOL = 1e-14    # ||K X - B|| / (||K|| ||X||), longdouble
LD_MAX_N = 1100         # longdouble LDL^T up to here, LAPACK + longdouble residual above

NRHS = [1, 2, 3, 4, 5, 8, 9, 17]  # leaf-solve groups: 1 | 2 | 4 | 4 | 8 | 8 | 2 x 8 | 3 x 8

DENSE_SHAPES = [
    (9, 2),      # r = 4 (uneven halves 4 / 5), then r = 2: gram_tn_small<4>, <2>
    (12, 3),     # r = 6, 3: <8>, <4>
    (14, 7),     # r = 7: <8>
    (16, 8),     # r = 8: 2r = 16, the last rank of the small-rank Gram kernel
    (17, 8),     # r = 8 over uneven halves 8 / 9
    (18, 9),     # r = 9: 2r = 18, the first rank of gram_tn_kernel
    (40, 5),     # r = 20, 10 (gram_tn_kernel) over 5 (<8>)
    (68, 8),     # r = 34, 17 (gram_tn_kernel) over 8 (<8>, at the switch)
    (2100, 1000),  # r = 1050: 2100 rows = two full 1024-row finalisation tiles and a 52-row one, 1050 columns each
]

LOWRANK_SHAPES = [
    (1025, 100),   # halves 512 / 513: a 1-row second tile
    (3073, 100),   # halves 1536 / 1537
    (4096, 1024),  # every node a multiple of 1024 rows (the aligned case)
    (5000, 100),   # six levels of ragged nodes, 2500 .. 156 rows
]


def _kernel():
    from george_b200 import kernels as K
    return 1.0 * K.ExpKernel(1.0)


def _inputs(n):
    rng = np.random.default_rng(7 + n)
    x = np.sort(rng.uniform(0, n / 50.0, n))[:, None]
    return x, 0.1 * np.ones(n)


class _Ref(object):
    def __init__(self, kernel, x, yerr):
        n = x.shape[0]
        self.n = n
        K = kernel.get_value(x)
        K[np.diag_indices(n)] += yerr ** 2
        self.K = K
        self.exact = n <= LD_MAX_N
        if self.exact:
            L, d = hiprec.ldlt_ld(K)
            assert np.all(d > 0)
            self.Lc = L * np.sqrt(d)[None, :]
            self.logdet = float(np.sum(np.log(d)))
            self.K_ld = K.astype(LD)
        else:
            self.cf = scipy.linalg.cho_factor(K, lower=True)
            self.logdet = float(2 * np.sum(np.log(np.diag(self.cf[0]))))
        rng = np.random.default_rng(n + 3)
        self.B = rng.normal(size=(n, sum(NRHS)))
        self.X = hiprec.solve_ld(self.Lc, self.B) if self.exact else scipy.linalg.cho_solve(self.cf, self.B)

    def residual(self, X, B):
        if self.exact:
            return hiprec.residual_ld(self.K_ld, X, B)
        return hiprec.residual_ld_blocked(self.K, X, B)


def _rel(X, Xr):
    Xr = np.asarray(Xr, dtype=LD)
    return float(np.sqrt(np.sum((np.asarray(X, dtype=LD) - Xr) ** 2) / np.sum(Xr ** 2)))


@pytest.fixture
def clean_env(monkeypatch):
    for var in ("BGP_SMALL_RANK_LIMIT", "BGP_LEAF_COLS", "BGP_NO_GRAPH", "BGP_NO_CULL", "BGP_LEAF_FACTOR"):
        monkeypatch.delenv(var, raising=False)
    return monkeypatch


def _run(n, min_size, exhaust, record_property):
    import george_b200 as george
    kernel = _kernel()
    x, yerr = _inputs(n)
    ref = _Ref(kernel, x, yerr)
    s = george.HODLRSolver(kernel, min_size=min_size, tol=1e-12, seed=42, rng_mode="pernode", exhaust=exhaust)
    s.compute(x, yerr)
    internal = [nd for nd in s.solver.nodes() if not nd["is_leaf"]]
    assert internal
    for nd in internal:  # the premise: K_h = K to rounding, with the intended ranks
        if exhaust == "dense":
            assert nd["rank"] == nd["half"], nd
        else:
            assert nd["rank"] == 1, nd

    logdet_err = abs(s.log_determinant - ref.logdet) / max(1.0, abs(ref.logdet))
    solve, resid = {}, {}
    offs = np.cumsum([0] + NRHS)
    for j, nrhs in enumerate(NRHS):
        B, Xr = ref.B[:, offs[j]:offs[j] + nrhs], ref.X[:, offs[j]:offs[j] + nrhs]
        X = s.apply_inverse(B)
        assert X.shape == (n, nrhs)
        solve[nrhs] = _rel(X, Xr)
        if ref.exact or nrhs in (1, 9):  # (O(n^2) longdouble per column)
            resid[nrhs] = ref.residual(X, B)
    y = ref.B[:, 0]
    q_ref = float(np.dot(y.astype(LD), np.asarray(ref.X[:, 0], dtype=LD)))
    solve["dot_solve"] = abs(s.dot_solve(y) - q_ref) / abs(q_ref)

    record_property("logdet_err", logdet_err)
    record_property("solve_err", max(solve.values()))
    record_property("residual_err", max(resid.values()))
    assert logdet_err <= LOGDET_TOL, logdet_err
    assert max(solve.values()) <= SOLVE_TOL, solve
    assert max(resid.values()) <= RESIDUAL_TOL, resid


@pytest.mark.parametrize("n,min_size", DENSE_SHAPES)
def test_level_ranks_around_the_small_gram_switch(gpu, clean_env, record_property, n, min_size):
    """Exact dense trees whose levels have r = 2 .. 1050: each small-rank Gram instantiation, r = 8 and 9 on either side
    of the switch, and levels of both kernels in one up-sweep."""
    _run(n, min_size, "dense", record_property)


@pytest.mark.parametrize("n,min_size", LOWRANK_SHAPES)
def test_rank_one_nodes_across_row_tiles(gpu, clean_env, record_property, n, min_size):
    """Rank-1 nodes of up to 2500 rows: the panel finalisation and the small-rank Gram product over 1024-row tiles, full
    and ragged."""
    _run(n, min_size, "lowrank", record_property)
