# -*- coding: utf-8 -*-
"""The ACA factors themselves (csrc/hodlr_kernels.cuh ``aca_kernel``, csrc/hodlr_aca2.cuh), read back through
``bgp_hodlr_node_factors``, against the algorithm they implement (hodlr.h:136-221) restated in longdouble.

For an internal node with left half L (columns) and right half R (rows), K12 = K[R, L] ~ Ur Vl^T with
Vl = the normalised residual rows (indexed by L) and Ur = the residual columns (indexed by R).  Checked here:

* normalisation: Vl[j_k, k] == 1 exactly and max |Vl[:, k]| <= 1 (the row residual is divided by its largest entry);
* interpolation: K12 - Ur Vl^T vanishes on every pivot row and column;
* the recursion itself, rerun in longdouble with the device's pivot sequence, and its stopping rule;
* the exhaustion claim of ``exhaust_mode = LOWRANK``: a node flagged ``dense_fallback`` has |K12 - Ur Vl^T| < 1e-14 on
  EVERY entry (with and without the bound culling of the candidate scan);
* the dense fill of ``exhaust_mode = DENSE``: Vl = I, Ur = K12;
* the HODLR matrix K_h assembled from the leaves and these factors: log-det and solves against its longdouble LDL^T.

Block sizes sit around the ACA's 1024-row work items (A2_CHUNK) and its 128-column culling groups.
"""
import numpy as np
import pytest

import hiprec

pytestmark = pytest.mark.gpu

LD = np.longdouble
EPS = np.finfo(np.float64).eps

# bars: 10-60x the largest value measured on one H100 80GB HBM3 (SXM, 400 W power limit)
INTERP_TOL = 5e-15     # max |K12 - Ur Vl^T| on the pivot rows / columns, / max|K12|              (measured 2.6e-16)
# The cross approximation along fixed pivots is K[:, J] K[I, J]^-1 K[I, :]; rounding on the cross is amplified by the
# conditioning of K[I, J] (its last pivots are ~1e-10 of max|K12|), so the float64 and longdouble products differ by
# far more than the interpolation error although both interpolate K on the cross to rounding.
RECURSION_TOL = 5e-8   # max |Ur Vl^T - (U V^T)_longdouble| / max|K12|                            (measured 3.3e-9)
EXHAUST_SLACK = 1e-15  # allowance above 1e-14 for the float64 rounding of the device's residual
#                        (measured: none needed, largest entry 9.7e-15)
DENSE_FILL_ULP = 1     # |Ur - K12| in units of the last place of K12                              (measured 0)
# K_h end to end.  K_h is the matrix the solver factorises, but for low-rank blocks the Woodbury matrices S are far less
# well conditioned than in the exact-K sweeps (test_gpu_hodlr_sweeps.py: solve 4.3e-13, residual 7.6e-16).  The
# largest values below are all from Matern-3/2, exhaust dense, tol 1e-10.
KH_LOGDET_TOL = 3e-12  # |logdet - ref| / max(1, |ref|)                                            (measured 2.3e-13)
# the forward error of a backward-stable solve is ~ cond(K_h) eps: the solve bar is scaled by the 2-norm condition number
KH_SOLVE_COND = 100.0  # ||X - X_ref|| / ||X_ref|| (and dot_solve) <= KH_SOLVE_COND cond(K_h) eps
#                        (measured 6.3: 3.2e-11 at cond 2.3e4, Matern-3/2, exhaust dense; cond up to 6.7e4)
KH_RESIDUAL_TOL = 1e-13  # ||K_h X - B|| / (||K_h|| ||X||)                                        (measured 7.3e-15)
KNIFE = 1e-6           # stopping-rule comparisons closer than this (relative) are not judged


def _kernel(kname):
    from george_b200 import kernels as K
    es2 = K.ExpSine2Kernel(gamma=1.0, log_period=np.log(3.0))
    return {"expsq_1d": 1.0 * K.ExpSquaredKernel(1.0),
            "m52_3d": 1.0 * K.Matern52Kernel(0.5, ndim=3),
            "cfg5_1d": 1.0 * K.ExpSquaredKernel(1.0) + 0.5 * es2,
            "prod_expsq_es2": 1.2 * K.ExpSquaredKernel(50.0) * es2,
            "m32_1d": 1.0 * K.Matern32Kernel(1.0)}[kname]


KNAMES = ["expsq_1d", "m52_3d", "cfg5_1d", "prod_expsq_es2", "m32_1d"]


def _tol(kname):
    return 1e-12 if kname == "m52_3d" else 1e-10


def _inputs(kname, n, seed=0):
    rng = np.random.default_rng(seed + n)
    if kname == "m52_3d":  # a slab, long along the split axis: node interfaces of ~1 x 1 keep the ranks moderate
        x = rng.uniform(0, 1, (n, 3)) * np.array([n / 100.0, 1.0, 1.0])
        return x[np.argsort(x[:, 0])]
    return np.sort(rng.uniform(0, 10.0 * n / 1000.0, n))[:, None]


# the root block is 1023, 1024, 1025 and 2049 columns wide (one A2_CHUNK work item -1, exactly, +1, two +1);
# min_size = N / 4 keeps the tree at two internal levels.  1001 / 60 has 15 internal nodes over four levels.
SHAPES = [(2046, 511), (2048, 512), (2050, 512), (4098, 1024), (1001, 60)]


def _compute(kname, n, min_size, rng_mode, exhaust, tol=None, yerr=0.1):
    from george_b200.solvers._hodlr import HODLRSolver
    kernel = _kernel(kname)
    x = _inputs(kname, n)
    s = HODLRSolver()
    s.compute(kernel, x, yerr * np.ones(n), min_size=min_size, tol=_tol(kname) if tol is None else tol, seed=42,
              rng_mode=rng_mode, exhaust=exhaust)
    return kernel, x, s


def _block(kernel, x, nd):
    lo, mid, hi = nd["start"], nd["start"] + nd["half"], nd["start"] + nd["size"]
    return kernel.get_value(x[mid:hi], x[lo:mid])  # K12 = K[right, left]


def _aca_ld(K12, rows, cols):
    """The recursion of hodlr.h:186-199 in longdouble along the given pivot sequence: (U, V, shortfall of each pivot
    below the largest entry of its residual row)."""
    nr, nc = K12.shape
    r = len(rows)
    U = np.zeros((nr, r), dtype=LD)
    V = np.zeros((nc, r), dtype=LD)
    short = np.zeros(r)
    for k in range(r):
        i, j = rows[k], cols[k]
        v = K12[i].astype(LD) - V[:, :k] @ U[i, :k]
        short[k] = float(np.max(np.abs(v)) - abs(v[j]))  # 0 if the pivot is the largest entry of the residual row
        V[:, k] = v / v[j]
        U[:, k] = K12[:, j].astype(LD) - U[:, :k] @ V[j, :k]
    return U, V, short


def _stopping_rule(Ur, Vl, tol, rank, max_rank, exhausted):
    """hodlr.h:203-214, evaluated on the device's own float64 factors (the quantities the device compared, up to the
    summation order): the rule must not fire before the final rank, and at the final rank it must have fired unless
    the rank hit min(rows, cols) or the rows ran out.  Comparisons within KNIFE (relative) are not judged.  Returns
    (judged steps before the last, 1 if the last step was judged)."""
    norm = 0.0
    tol2 = tol * tol
    judged = 0
    for k in range(rank):
        rowcol = float(np.dot(Ur[:, k], Ur[:, k]) * np.dot(Vl[:, k], Vl[:, k]))
        last = k == rank - 1
        if k + 1 >= max_rank:
            assert last
            return judged, 0
        fired = rowcol < tol2 * norm
        if abs(rowcol - tol2 * norm) > KNIFE * tol2 * norm:
            if not last:
                assert not fired, (k, rank, rowcol, tol2 * norm)
                judged += 1
            elif not exhausted:
                assert fired, (k, rank, rowcol, tol2 * norm)
                return judged, 1
        if last:
            return judged, 0
        norm += rowcol
        if k > 0:
            norm += 2 * float(np.max(np.abs(Ur[:, :k].T @ Ur[:, k]))) + 2 * float(np.max(np.abs(Vl[:, :k].T @ Vl[:, k])))
    return judged, 0


def _max_abs_residual_ld(K12, Ur, Vl, rows=256):
    worst = 0.0
    VlT = Vl.astype(LD).T
    for i0 in range(0, K12.shape[0], rows):
        R = K12[i0:i0 + rows].astype(LD) - Ur[i0:i0 + rows].astype(LD) @ VlT
        worst = max(worst, float(np.max(np.abs(R))))
    return worst


@pytest.mark.parametrize("exhaust", ["lowrank", "dense"])
@pytest.mark.parametrize("rng_mode", ["pernode", "reference"])
@pytest.mark.parametrize("n,min_size", SHAPES)
@pytest.mark.parametrize("kname", KNAMES)
def test_aca_factors(gpu, monkeypatch, record_property, kname, n, min_size, rng_mode, exhaust):
    monkeypatch.delenv("BGP_NO_CULL", raising=False)
    kernel, x, s = _compute(kname, n, min_size, rng_mode, exhaust)
    tol = _tol(kname)
    worst = {"interp": 0.0, "recursion": 0.0, "exhaust": 0.0, "dense_ulp": 0.0}
    judged_steps = judged_final = rule_final = 0  # stopping-rule decisions judged; nodes that stopped on the rule
    fallback_nodes = []
    for idx, nd in enumerate(s.nodes()):
        if nd["is_leaf"]:
            continue
        rank = nd["rank"]
        Vl, Ur = s.factors(idx)
        assert Vl.shape == (nd["half"], rank) and Ur.shape == (nd["size"] - nd["half"], rank)
        K12 = _block(kernel, x, nd)
        kmax = float(np.max(np.abs(K12)))
        if nd["dense_fallback"] and exhaust == "dense":
            # hodlr.h:161-176: V = I, U = the block (n_cols <= n_rows always: half = size / 2)
            assert rank == nd["half"]
            assert np.array_equal(Vl, np.eye(rank))
            ulp = np.abs(Ur - K12) / np.spacing(np.abs(K12))
            worst["dense_ulp"] = max(worst["dense_ulp"], float(np.max(ulp)))
            assert np.max(ulp) <= DENSE_FILL_ULP, (idx, float(np.max(ulp)))
            continue
        if rank == 0:
            assert nd["dense_fallback"] and kmax < 1e-14
            continue
        rows, cols = s.pivots(idx, rank)
        # normalisation: bit-exact
        assert np.all(Vl[cols, np.arange(rank)] == 1.0), idx
        assert np.max(np.abs(Vl)) <= 1.0, idx
        # interpolation on the pivot rows and columns
        Rr = K12[rows].astype(LD) - Ur[rows].astype(LD) @ Vl.astype(LD).T
        Rc = K12[:, cols].astype(LD) - Ur.astype(LD) @ Vl[cols].astype(LD).T
        interp = max(float(np.max(np.abs(Rr))), float(np.max(np.abs(Rc)))) / kmax
        worst["interp"] = max(worst["interp"], interp)
        # the recursion in longdouble along the same pivots.  Compare the products: single columns can be amplified by a
        # small pivot.  P_dev - P_ld = (Ur - U) Vl^T + U (Vl - V)^T, the differences rounded only after the subtraction.
        U, V, _ = _aca_ld(K12, rows, cols)
        dU = (Ur.astype(LD) - U).astype(np.float64)
        dV = (Vl.astype(LD) - V).astype(np.float64)
        rec = float(np.max(np.abs(dU @ Vl.T + U.astype(np.float64) @ dV.T))) / kmax
        worst["recursion"] = max(worst["recursion"], rec)
        jn, jl = _stopping_rule(Ur, Vl, tol, rank, min(Ur.shape[0], Vl.shape[0]), bool(nd["dense_fallback"]))
        judged_steps += jn
        judged_final += jl
        if not nd["dense_fallback"] and rank < min(Ur.shape[0], Vl.shape[0]):
            rule_final += 1
        if nd["dense_fallback"]:
            fallback_nodes.append((idx, K12))
    if exhaust == "lowrank":
        # the exhaustion claim, with the culled candidate scan (above) and the exhaustive one
        for cull in (True, False):
            if not cull:
                monkeypatch.setenv("BGP_NO_CULL", "1")
                kernel, x, s = _compute(kname, n, min_size, rng_mode, exhaust)
                fallback_nodes = [(i, _block(kernel, x, nd)) for i, nd in enumerate(s.nodes())
                                  if not nd["is_leaf"] and nd["dense_fallback"] and nd["rank"] > 0]
            for idx, K12 in fallback_nodes:
                Vl, Ur = s.factors(idx)
                worst["exhaust"] = max(worst["exhaust"], _max_abs_residual_ld(K12, Ur, Vl))
    for k, v in worst.items():
        record_property(k, v)
    record_property("rule_steps_judged", judged_steps)
    record_property("rule_final_judged", judged_final)
    record_property("rule_final_nodes", rule_final)
    assert worst["interp"] <= INTERP_TOL, worst
    assert worst["recursion"] <= RECURSION_TOL, worst
    assert worst["exhaust"] < 1e-14 + EXHAUST_SLACK, worst


def test_node_factors_errors(gpu):
    """The export refuses leaves, out-of-range nodes and a handle that was never computed."""
    from george_b200 import _lib
    from george_b200.solvers._hodlr import HODLRSolver
    HODLRSolver.release_parked()
    s = HODLRSolver()
    buf = np.zeros(16)
    assert s._lib.bgp_hodlr_node_factors(s._ptr, 0, _lib.ptr(buf)) == _lib.BGP_ERR_NOT_COMPUTED
    _, _, s = _compute("m32_1d", 300, 60, "pernode", "lowrank")
    nodes = s.nodes()
    leaf = next(i for i, nd in enumerate(nodes) if nd["is_leaf"])
    for bad in (leaf, -1, len(nodes)):
        assert s._lib.bgp_hodlr_node_factors(s._ptr, bad, _lib.ptr(buf)) == _lib.BGP_ERR_INDEX
    with pytest.raises(IndexError):
        s.factors(leaf)
    Vl, Ur = s.factors(0)
    assert Vl.shape[1] == Ur.shape[1] == nodes[0]["rank"] > 0


KH_CASES = [("pernode", "lowrank", None, 0.1), ("reference", "dense", None, 0.1), ("reference", "dense", 0.1, 5.0)]


@pytest.mark.parametrize("rng_mode,exhaust,tol,yerr", KH_CASES)
@pytest.mark.parametrize("kname", KNAMES)
def test_hodlr_matrix_end_to_end(gpu, monkeypatch, record_property, kname, rng_mode, exhaust, tol, yerr):
    """K_h assembled from the leaves (K blocks + yerr^2) and the exported factors IS the matrix the solver factorises:
    log-det, solves and dot_solve against a longdouble LDL^T of K_h, at float64 rounding, including the reference's
    default tol = 0.1 (yerr = 5 keeps that K_h positive definite: at yerr = 1 the Matern-5/2 one is not)."""
    monkeypatch.delenv("BGP_NO_CULL", raising=False)
    n, min_size = 1001, 60
    kernel, x, s = _compute(kname, n, min_size, rng_mode, exhaust, tol=tol, yerr=yerr)
    Kh = kernel.get_value(x)
    Kh[np.diag_indices(n)] += yerr ** 2
    for idx, nd in enumerate(s.nodes()):
        if nd["is_leaf"]:
            continue
        lo, mid, hi = nd["start"], nd["start"] + nd["half"], nd["start"] + nd["size"]
        Vl, Ur = s.factors(idx)
        P = (Ur.astype(LD) @ Vl.astype(LD).T).astype(np.float64)
        Kh[mid:hi, lo:mid] = P
        Kh[lo:mid, mid:hi] = P.T
    cond = float(np.linalg.cond(Kh))
    L, d = hiprec.ldlt_ld(Kh)
    assert np.all(d > 0), "K_h is not positive definite"
    Lc = L * np.sqrt(d)[None, :]
    ld_ref = float(np.sum(np.log(d)))
    ld_err = abs(s.log_determinant - ld_ref) / max(1.0, abs(ld_ref))
    rng = np.random.default_rng(n)
    B = rng.normal(size=(n, 9))
    X = s.apply_inverse(B)
    Xr = hiprec.solve_ld(Lc, B)
    sol = float(np.sqrt(np.sum((X.astype(LD) - Xr) ** 2) / np.sum(Xr ** 2)))
    res = hiprec.residual_ld(Kh, X, B)
    y = B[:, 0]
    q_ref = float(np.dot(y.astype(LD), Xr[:, 0]))
    sol = max(sol, abs(s.dot_solve(y) - q_ref) / abs(q_ref))
    record_property("logdet_err", ld_err)
    record_property("solve_err", sol)
    record_property("cond", cond)
    record_property("solve_over_cond_eps", sol / (cond * EPS))
    record_property("residual_err", res)
    assert ld_err <= KH_LOGDET_TOL
    assert sol <= KH_SOLVE_COND * cond * EPS, (sol, cond)
    assert res <= KH_RESIDUAL_TOL
