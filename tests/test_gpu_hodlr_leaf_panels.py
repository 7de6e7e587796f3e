# -*- coding: utf-8 -*-
"""The leaf LDL^T kernel (``leaf_factor_kernel``, csrc/hodlr_leaf.cuh) at its internal block boundaries, against the
extended-precision reference and against ``leaf_build_factor_kernel`` (``BGP_LEAF_FACTOR=generic``).

The kernel works in 32-column panels, updates each panel in 16-row tiles and solves the rows below a panel's diagonal
block one per thread of 256, so the sizes below sit on either side of 16, 32, 64, 128 and 256 rows and of the 288- and
544-row leaves where a thread takes a second and a third row.  ``m32_1d`` runs the Matern-3/2 evaluator specialised for
1-D inputs, ``sum3d`` the general interpreter on 3-D inputs.
"""
import pytest

from test_gpu_hodlr_leaves import LOGDET_TOL, SOLVE_TOL, _check_exact_solver, _problem, _rel

pytestmark = pytest.mark.gpu

PANEL_N = [15, 16, 17, 63, 64, 65, 127, 128, 129, 255, 256, 257, 288, 289, 545]


@pytest.mark.parametrize("n", PANEL_N)
@pytest.mark.parametrize("kname", ["m32_1d", "sum3d"])
def test_single_leaf_at_panel_boundaries_is_exact_ldlt(gpu, monkeypatch, record_property, kname, n):
    from george_b200.solvers._hodlr import HODLRSolver
    monkeypatch.delenv("BGP_LEAF_FACTOR", raising=False)
    monkeypatch.delenv("BGP_LEAF_COLS", raising=False)
    kernel, x, yerr, K, Lc = _problem(kname, n)
    s = HODLRSolver()
    s.compute(kernel, x, yerr, min_size=n, tol=1e-12, seed=42)
    nodes = s.nodes()
    assert len(nodes) == 1 and nodes[0]["is_leaf"]
    _check_exact_solver(s, K, Lc, [1, 9], n, record_property)


@pytest.mark.parametrize("m", [1, 33, 100, 257, 768])
def test_generic_and_tensor_leaf_factor_agree_on_the_interpreter(gpu, monkeypatch, m):
    """An N-D program runs the interpreter in both kernels: both LDL^T implementations against the reference and
    against each other."""
    from george_b200.solvers._hodlr import HODLRSolver
    monkeypatch.delenv("BGP_LEAF_COLS", raising=False)
    kernel, x, yerr, K, Lc = _problem("sum3d", m)
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
