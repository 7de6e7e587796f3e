# -*- coding: utf-8 -*-
"""The leaf LDL^T kernel's one-panel lookahead (``leaf_factor_kernel``, csrc/hodlr_leaf.cuh) at its edges.

While one warp factorises the diagonal block of panel p, the other warps evaluate panel p + 1 and accumulate its update
from the columns before panel p; both are parked in the leaf's block of the factor buffer and picked up at the next
panel.  The sizes below sit on either side of one panel (32 rows), two panels and the 256-row leaf, with a partial last
panel in every odd size; 700 and 768 rows are the largest leaves with many panels in flight.  ``m32_1d`` runs the
Matern-3/2 evaluator specialised for 1-D inputs, ``sum3d`` the general interpreter on 3-D inputs, and ``expsq_1d`` the
ExpSquared leaves of the benchmark's cfg2 (its point density and noise), the ill-conditioned ones: cond(K) is 1.1e4 at
128 rows and 2.3e4 at 768.

The lookahead keeps every entry's summation order: the parked accumulators are continued with the panel's own columns
before the one subtraction, as the panel-by-panel schedule did.  So the factor, D and the log-determinant equal those
of the panel-by-panel kernel bit for bit; ``tests/golden/leaf_factor_bits.npz`` holds that kernel's log-determinant,
solves and symmetric-factor products for every case (``tests/golden/make_golden_leaf_factor.py``).
"""
import os

import numpy as np
import pytest

import hiprec
from test_gpu_hodlr_leaves import LOGDET_TOL, RESIDUAL_TOL, SOLVE_TOL, _problem, _rel, _solve_ref

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "leaf_factor_bits.npz")

LOOKAHEAD_N = [1, 31, 32, 33, 63, 64, 65, 255, 256, 257, 700, 768]
CASES = ([("m32_1d", n) for n in LOOKAHEAD_N] + [("sum3d", n) for n in (1, 33, 65, 257, 768)] +
         [("expsq_1d", n) for n in (33, 128, 257, 768)])

_CACHE = {}


def leaf_problem(kname, n):
    """(kernel, x, yerr, K, Lc): Lc a longdouble Cholesky factor of K (every n here is <= 800)."""
    if kname != "expsq_1d":
        return _problem(kname, n)
    if n not in _CACHE:
        from george_b200 import kernels as K
        kernel = 1.0 * K.ExpSquaredKernel(1.0)
        rng = np.random.default_rng(n)
        x = np.sort(rng.uniform(0, 10 * n / 1000, n))[:, None]
        yerr = 0.1 * np.ones(n)
        Km = kernel.get_value(x)
        Km[np.diag_indices(n)] += yerr ** 2
        L, d = hiprec.ldlt_ld(Km)
        _CACHE[n] = (kernel, x, yerr, Km, L * np.sqrt(d)[None, :])
    return _CACHE[n]


def leaf_outputs(s, n):
    """What a single-leaf factorisation gives that depends on every bit of L and D: the log-determinant, two solves
    and the symmetric factor L D^1/2 applied to a vector."""
    rng = np.random.default_rng(1000 + n)
    B = rng.normal(size=(n, 2))
    z = rng.normal(size=n)
    return {"logdet": np.array([s.log_determinant]), "solve": s.apply_inverse(B),
            "sym": s.apply_symmetric_factor(z)}


def single_leaf(kname, n):
    from george_b200.solvers._hodlr import HODLRSolver
    kernel, x, yerr, K, Lc = leaf_problem(kname, n)
    s = HODLRSolver()
    s.compute(kernel, x, yerr, min_size=n, tol=1e-12, seed=42)
    nodes = s.nodes()
    assert len(nodes) == 1 and nodes[0]["is_leaf"]
    return s, kernel, x, yerr, K, Lc


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


@pytest.fixture(autouse=True)
def _default_leaf_paths(monkeypatch):
    monkeypatch.delenv("BGP_LEAF_FACTOR", raising=False)
    monkeypatch.delenv("BGP_LEAF_COLS", raising=False)


@pytest.mark.parametrize("kname,n", CASES)
def test_lookahead_leaf_is_exact_ldlt(gpu, record_property, kname, n):
    """Against the longdouble LDL^T at the leaf tests' bars.  The forward-error bar is stated for cond(K) <~ 1e4; the
    ill-conditioned ExpSquared leaves get it scaled by cond(K) / 1e4."""
    s, kernel, x, yerr, K, Lc = single_leaf(kname, n)
    cond = float(np.linalg.cond(K))
    ld_ref = float(hiprec.logdet_ld(Lc))
    ld_err = abs(s.log_determinant - ld_ref) / max(1.0, abs(ld_ref))
    B = np.random.default_rng(7 * n).normal(size=(n, 9))
    X = s.apply_inverse(B)
    fwd = _rel(X, _solve_ref(Lc, B))
    res = hiprec.residual_ld(K, X, B)
    for name, v in (("cond", cond), ("logdet_err", ld_err), ("solve_err", fwd), ("residual_err", res)):
        record_property(name, v)
    assert ld_err <= LOGDET_TOL, ld_err
    assert fwd <= SOLVE_TOL * max(1.0, cond / 1e4), (fwd, cond)
    assert res <= RESIDUAL_TOL, res


@pytest.mark.parametrize("kname,n", CASES)
def test_lookahead_factor_equals_panel_by_panel_bits(gpu, kname, n):
    """Two computes on one handle give the same bits, and those are the panel-by-panel kernel's."""
    golden = np.load(GOLDEN)
    s = single_leaf(kname, n)[0]
    first = leaf_outputs(s, n)
    s.compute(*leaf_problem(kname, n)[:3], min_size=n, tol=1e-12, seed=42)
    second = leaf_outputs(s, n)
    for key in ("logdet", "solve", "sym"):
        assert np.array_equal(_bits(first[key]), _bits(second[key])), key
        ref = golden["{0}_{1}_{2}".format(kname, n, key)]
        assert np.array_equal(_bits(first[key]), _bits(ref)), (key, _rel(first[key], ref))
