# -*- coding: utf-8 -*-
"""The HODLR symmetric factor K~ = W W^T (csrc/hodlr_sym.cu, csrc/hodlr_sym.cuh) at its block, chunk and staging
boundaries, against exact or extended-precision references.

* ``c * ExpKernel(m)`` on sorted 1-D points with ``yerr = 0`` is an Ornstein-Uhlenbeck covariance whose Cholesky factor
  L is known entry by entry (``ou_reference.OU``), with L^-1 z an O(n) longdouble sweep.  Its off-diagonal blocks are
  exactly rank 1, so
  - with ``exhaust="dense"`` every internal node runs out of rows and stores its block exactly, rank = half: K~ = K and
    the level ranks are set by N and min_size (``tests/test_gpu_hodlr_sweeps.py``).  Those columns are numerically
    dependent, so the bases come from the Householder path;
  - with ``exhaust="lowrank"`` every internal node has rank 1: K~ = K to rounding at any N.
  For any symmetric factor of K, E = L^-1 W is orthogonal, so max |E^T E - I| (on the identity, or on a random block Z
  as (E Z)^T (E Z) - Z^T Z) measures W directly; a root that is one leaf has W = L, compared entry by entry.
* General kernels (``exhaust="lowrank"``, CholeskyQR3 bases): W (W^T Z) against K~ Z accumulated in longdouble from
  the leaf blocks and the nodes' ACA factors, and log|K~| against a longdouble L D L^T of the assembled K~.
* ``BGP_SYM_QR=householder`` puts every node through the Householder QR; W is unique when the bases have full column
  rank, so the two factors agree entry by entry, to within the conditioning of the ACA's bases (QR_TOL).

Boundaries reached: ranks across sym_tn's 32-column Q tiles, above the 256 threads of sym_qr_pass_kernel and past
the former 800 staging cliff of sym_nn_kernel; zero-padded columns; hundreds of ancestor columns; half-nodes across
the 2048-row chunks of the partial products; leaves over 3200 rows (the 1-column leaf kernels) and around 256 rows;
apply widths across the 8-column leaf groups and the 64-column apply groups; levels of 32768 and 65536 nodes.
"""
import numpy as np
import pytest

import hiprec
from ou_reference import OU, exp_problem

pytestmark = pytest.mark.gpu

LD = np.longdouble

# Bars: 10-60x the largest value measured on one H100 80GB HBM3 (SXM, 700 W power limit), never looser than the
# factor's targets, except QR_TOL (below).
ORTH_TOL = 1e-13      # max |E^T E - I| or max |(E Z)^T (E Z) - Z^T Z| / max |Z^T Z|, E = L^-1 W  (measured 3.2e-15)
ADJ_TOL = 3e-15       # |z1 . W z2 - W^T z1 . z2| / sum |z1_i (W z2)_i|, longdouble                (measured 1.3e-16)
LOGDET_TOL = 1e-13    # |symmetric_log_determinant - OU log|K|| / |log|K||, also the solver's     (measured 7.7e-15)
LDLT_TOL = 2e-14      # |symmetric_log_determinant - longdouble L D L^T of K~| / |ref|             (measured 8.7e-16)
CHOL_TOL = 1e-14      # root leaf: max |W[:, j] - L[:, j]| / max |L[:, j]|, also rows of W^T       (measured 8.2e-16)
KZ_TOL = 1e-15        # ||W (W^T Z) - K~ Z||_F / (||K~||_F ||Z||_F), K~ Z in longdouble, both QRs  (measured 5.2e-17)
SOLVE_TOL = 5e-15     # apply_inverse against the OU closed form, relative 2-norm                   (measured 2.6e-16)
# max |W Z (CholeskyQR3) - W Z (Householder)| / max |W Z|.  W is unique for bases of full column rank, but it moves
# with the bases by about cond(V_h) u, and the ACA's columns at tol = 1e-12 are far from orthogonal: measured 2.3e-15
# (Matern-3/2, rank 2), 5.2e-14 (1-D ExpSquared), 2.8e-14 (2-D, rank 481) and 1.5e-12 (2-D, ranks 38-79, N = 4096).
# W W^T from either path meets KZ_TOL, which is the property sampling needs.
QR_TOL = 2e-11

IDENT_MAX = 4096      # W applied to the identity up to here, to a random 130-column block above
SY_MAX_RANK = 2048    # the symmetric factor's rank limit (csrc/hodlr_sym.cu)


@pytest.fixture
def env(monkeypatch):
    for var in ("BGP_SYM_QR", "BGP_SMALL_RANK_LIMIT", "BGP_LEAF_COLS", "BGP_NO_GRAPH", "BGP_NO_CULL",
                "BGP_LEAF_FACTOR"):
        monkeypatch.delenv(var, raising=False)
    return monkeypatch


# ---- references ----------------------------------------------------------------------------------------------------

def _gram(A):
    """A^T A for an (n, k) float64 or longdouble A, well below float64 rounding: A = hi + lo in float64, the products
    taken in float64 over 1024-row blocks and the blocks summed in longdouble."""
    A = np.asarray(A)
    hi = A.astype(np.float64)
    lo = (A.astype(LD) - hi).astype(np.float64)
    G = np.zeros((A.shape[1], A.shape[1]), dtype=LD)
    for i0 in range(0, A.shape[0], 1024):
        h, l = hi[i0:i0 + 1024], lo[i0:i0 + 1024]
        G += (h.T @ h).astype(LD)
        G += (h.T @ l + l.T @ h).astype(LD)
    return G


def _chol_rows(ou, rows):
    """``L[rows, :]`` of the OU factor (``(len(rows), n)``), entry by entry."""
    out = np.zeros((len(rows), ou.n), dtype=LD)
    for k, j in enumerate(rows):
        out[k, :j + 1] = ou.sqrtc * ou.s[:j + 1] * np.exp(-(ou.x[j] - ou.x[:j + 1]) / ou.ell)
    return out


def _relmax(a, ref):
    ref = np.asarray(ref, dtype=LD)
    return float(np.max(np.abs(np.asarray(a, dtype=LD) - ref)) / np.max(np.abs(ref)))


def _ou_solver(n, min_size, exhaust, seed=None):
    from george_b200 import kernels
    from george_b200.solvers._hodlr import HODLRSolver
    c, m = 1.0, 1.0
    x = exp_problem(n, np.sqrt(m), seed=n if seed is None else seed)
    s = HODLRSolver()
    s.compute(c * kernels.ExpKernel(m), x[:, None], np.zeros(n), min_size=min_size, tol=1e-12, seed=42,
              rng_mode="pernode", exhaust=exhaust)
    return s, OU(x, c, m)


def _internal(s):
    return [d for d in s.nodes() if not d["is_leaf"]]


def _level_ranks(s):
    ranks = {}
    for d in _internal(s):
        ranks.setdefault(d["depth"], set()).add(d["rank"])
    return ranks


def _check_ou(s, ou, record_property, seed=0, ident_max=IDENT_MAX):
    """E^T E = I, the adjoint identity, log|K~| against the closed form and reproducible applies; returns the errors."""
    n = ou.n
    rng = np.random.default_rng(seed)
    errs = {}
    if n <= ident_max:
        W = s.apply_symmetric_factor(np.eye(n))
        E = ou.inv_chol(W)
        errs["orth"] = float(np.max(np.abs(_gram(E) - np.eye(n, dtype=LD))))
        Z = np.eye(n)[:, rng.choice(n, min(n, 9), replace=False)]
        Y = s.apply_symmetric_factor(Z)
    else:
        Z = rng.standard_normal((n, 130))
        Y = s.apply_symmetric_factor(Z)
        GZ = _gram(Z)
        errs["orth"] = float(np.max(np.abs(_gram(ou.inv_chol(Y)) - GZ)) / np.max(np.abs(GZ)))
    assert np.array_equal(s.apply_symmetric_factor(Z), Y)  # the same factorisation applies with the same bits
    z1, z2 = rng.standard_normal(n), rng.standard_normal(n)
    wz2 = s.apply_symmetric_factor(z2).astype(LD)
    wtz1 = s.apply_symmetric_factor(z1, transpose=True).astype(LD)
    a, b = np.sum(z1.astype(LD) * wz2), np.sum(wtz1 * z2.astype(LD))
    errs["adjoint"] = float(abs(a - b) / np.sum(np.abs(z1.astype(LD) * wz2)))
    ref = ou.logdet()
    errs["logdet"] = float(abs(LD(s.symmetric_log_determinant) - ref) / abs(ref))
    for k, v in errs.items():
        record_property(k, v)
    assert errs["orth"] <= ORTH_TOL, errs
    assert errs["adjoint"] <= ADJ_TOL, errs
    assert errs["logdet"] <= LOGDET_TOL, errs
    return errs


# ---- 1./2. ranks on exact dense trees ------------------------------------------------------------------------------

DENSE_SHAPES = [
    (3, 1),                    # rank 1 over a size-2 node
    (62, 31), (64, 32), (66, 33),  # around sym_tn's 32-column Q tiles
    (130, 65),                 # 65: three tiles, the last of one column
    (258, 129),                # 129
    (510, 255), (512, 64), (514, 257),  # around the 256 threads of the per-column loops; (512, 64): 256, 128, 64
    (1001, 60),                # ranks 500, 250, 125, then 62 and 63 in one level (zero-padded columns)
    (1024, 32),                # ranks 512 .. 32: 960 ancestor columns over every leaf
    (1598, 799),               # the largest rank sym_nn_kernel staged 32 rows of before the rows were sized from r
    (1600, 800),               # 800: formerly rejected
    (2048, 1024),              # 1024
]


@pytest.mark.parametrize("n,min_size", DENSE_SHAPES)
def test_dense_tree_ranks(gpu, env, record_property, n, min_size):
    s, ou = _ou_solver(n, min_size, "dense")
    internal = _internal(s)
    assert internal and all(d["rank"] == d["half"] for d in internal)  # every block stored exactly: K~ = K
    ranks = _level_ranks(s)
    record_property("level_ranks", str(sorted((k, sorted(v)) for k, v in ranks.items())))
    if (n, min_size) == (1001, 60):
        assert ranks[3] == {62, 63}
    _check_ou(s, ou, record_property)
    record_property("build_ms", s.symmetric_factor_timing()["build_ms"])


def test_rank_above_the_limit_is_rejected_before_any_launch(gpu, env):
    from george_b200 import _lib
    n = 2 * (SY_MAX_RANK + 1)
    s, ou = _ou_solver(n, SY_MAX_RANK + 1, "dense")
    assert s.nodes()[0]["rank"] == SY_MAX_RANK + 1
    lib = _lib.load()
    before = lib.bgp_launch_count()
    msg = r"node 0 \(rows \[0, {0}\), level 0\) has rank {1}, above the symmetric factor's limit of {2}".format(
        n, SY_MAX_RANK + 1, SY_MAX_RANK)
    with pytest.raises(ValueError, match=msg):
        s.symmetric_log_determinant
    with pytest.raises(ValueError, match=msg):
        s.apply_symmetric_factor(np.ones(n))
    assert lib.bgp_launch_count() == before
    # the factorisation itself is untouched
    assert abs(s.log_determinant - float(ou.logdet())) <= 1e-12 * abs(float(ou.logdet()))


# ---- 3. chunk boundaries of the partial products -------------------------------------------------------------------

CHUNK_SHAPES = [
    (4094, 200), (4096, 200), (4098, 200),  # half-nodes of 2047, 2048 and 2049 rows around one 2048-row chunk
    (8192, 300), (8194, 300),               # 4096 (two full chunks), 4097
    (12290, 300),                           # 6145: three chunks and one row
    (262144, 256),                          # the at-scale shape: 10 levels, halves of 131072 rows (64 chunks)
]


@pytest.mark.parametrize("n,min_size", CHUNK_SHAPES)
def test_chunk_boundaries(gpu, env, record_property, n, min_size):
    s, ou = _ou_solver(n, min_size, "lowrank")
    nodes = s.nodes()
    assert {d["rank"] for d in nodes if not d["is_leaf"]} == {1}
    root = nodes[0]
    record_property("root_halves", str((root["half"], root["size"] - root["half"])))
    assert root["size"] - root["half"] == n - n // 2
    _check_ou(s, ou, record_property, seed=n)


# ---- 4. leaf staging -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [3200, 3201, 5000])
def test_root_leaf_is_the_cholesky_factor(gpu, env, record_property, n):
    """A root that is one leaf: W = L D^1/2 = L.  3200 rows stage 8 columns per CTA; 3201 and 5000 take the 1-column
    kernels (sym_leaf_product_kernel<1>, both directions)."""
    s, ou = _ou_solver(n, n, "lowrank")
    assert len(s.nodes()) == 1 and s.nodes()[0]["is_leaf"]
    rng = np.random.default_rng(n)
    cols = sorted({0, 1, 2, 7, 8, 9, 31, 32, 255, 256, 257, n // 2, n - 9, n - 8, n - 2, n - 1}
                  | set(rng.choice(n, 20, replace=False).tolist()))
    Z = np.eye(n)[:, cols]
    Wc = s.apply_symmetric_factor(Z)
    Lc = ou.chol_columns(cols)
    col_err = max(_relmax(Wc[:, k], Lc[:, k]) for k in range(len(cols)))
    Wr = s.apply_symmetric_factor(Z, transpose=True)  # W^T e_j = row j of L
    Lr = _chol_rows(ou, cols)
    row_err = max(_relmax(Wr[:, k], Lr[k]) for k in range(len(cols)))
    ld_err = float(abs(LD(s.symmetric_log_determinant) - ou.logdet()) / abs(ou.logdet()))
    record_property("col_err", col_err)
    record_property("row_err", row_err)
    record_property("logdet", ld_err)
    assert col_err <= CHOL_TOL and row_err <= CHOL_TOL and ld_err <= LOGDET_TOL


@pytest.mark.parametrize("n,min_size", [
    (7000, 2000),               # two 3500-row leaves: sym_leaf_forward_kernel<1> over the root's column
    (1020, 255), (1024, 256), (1028, 257),  # leaves of 255, 256 and 257 rows around the 256-thread loops
])
def test_leaf_staging(gpu, env, record_property, n, min_size):
    s, ou = _ou_solver(n, min_size, "lowrank")
    leaves = [d["size"] for d in s.nodes() if d["is_leaf"]]
    record_property("leaf_sizes", str(sorted(set(leaves))))
    assert max(leaves) == n // (4 if min_size < 1000 else 2)
    assert {d["rank"] for d in _internal(s)} == {1}
    _check_ou(s, ou, record_property, seed=n)


# ---- 5./6. general kernels on the CholeskyQR path, and against the Householder path ------------------------------

def _general(name):
    from george_b200 import kernels as K
    return {
        "m32": (1.0 * K.Matern32Kernel(1.0), 1),
        "expsq": (1.0 * K.ExpSquaredKernel(1.0), 1),
        "general2d": (1.0 * K.ExpSquaredKernel([[4.0, 0.6], [0.6, 2.0]], ndim=2), 2),
        # a short length scale: the root's block has a numerical rank near 300 at tol = 1e-12
        "general2d_short": (1.0 * K.ExpSquaredKernel([[0.12, 0.018], [0.018, 0.06]], ndim=2), 2),
    }[name]


def _points(n, ndim, seed=3):
    rng = np.random.default_rng(seed)
    if ndim == 1:
        return np.sort(rng.uniform(0, 10 * n / 1000, n))[:, None]
    x = rng.uniform(0, 4, (n, 2))
    return x[np.argsort(x[:, 0])]


def _ktilde_apply(s, kernel, x, yerr, Z):
    """(K~ Z in longdouble, ||K~||_F): the exact leaf blocks and Ur Vl^T / Vl Ur^T of every internal node."""
    Zl = np.asarray(Z, dtype=LD)
    out = np.zeros_like(Zl)
    fro2 = 0.0
    for i, nd in enumerate(s.nodes()):
        a, m, h = nd["start"], nd["size"], nd["half"]
        if nd["is_leaf"]:
            K = kernel.get_value(x[a:a + m]) + np.diag(yerr[a:a + m] ** 2)
            out[a:a + m] += np.einsum("ij,jk->ik", K.astype(LD), Zl[a:a + m])
            fro2 += float(np.sum(K * K))
        elif nd["rank"] > 0:
            Vl, Ur = s.factors(i)  # K~[right, left] = Ur Vl^T
            Vl_, Ur_ = Vl.astype(LD), Ur.astype(LD)
            out[a + h:a + m] += np.einsum("ij,jk->ik", Ur_, np.einsum("ji,jk->ik", Vl_, Zl[a:a + h]))
            out[a:a + h] += np.einsum("ij,jk->ik", Vl_, np.einsum("ji,jk->ik", Ur_, Zl[a + h:a + m]))
            fro2 += 2 * float(np.sum((Ur.T @ Ur) * (Vl.T @ Vl)))
    return out, np.sqrt(fro2)


def _assemble(s, kernel, x, yerr):
    n = x.shape[0]
    K = kernel.get_value(x) + np.diag(yerr ** 2)
    Kt = np.zeros((n, n))
    for i, nd in enumerate(s.nodes()):
        a, m, h = nd["start"], nd["size"], nd["half"]
        if nd["is_leaf"]:
            Kt[a:a + m, a:a + m] = K[a:a + m, a:a + m]
        elif nd["rank"] > 0:
            Vl, Ur = s.factors(i)
            B = Ur @ Vl.T
            Kt[a + h:a + m, a:a + h] = B
            Kt[a:a + h, a + h:a + m] = B.T
    return Kt


GENERAL_CASES = [
    ("m32", 1000, 64),               # rank 2
    ("expsq", 1000, 64),
    ("general2d", 1000, 64),         # ranks across 32
    ("expsq", 4098, 128),            # halves of 2049 rows
    ("general2d", 4096, 256),        # halves of 2048 rows, ranks across 32
    ("general2d_short", 2048, 256),  # a level rank above 256: sym_qr_pass_kernel's per-column loops wrap
]


@pytest.mark.parametrize("name,n,min_size", GENERAL_CASES)
def test_general_kernels_cholesky_qr_and_householder(gpu, env, record_property, name, n, min_size):
    from george_b200.solvers._hodlr import HODLRSolver
    kernel, ndim = _general(name)
    x = _points(n, ndim)
    yerr = 0.1 + 0.05 * np.random.default_rng(1).uniform(size=n)
    kw = dict(min_size=min_size, tol=1e-12, seed=42, rng_mode="pernode", exhaust="lowrank")
    s = HODLRSolver()
    s.compute(kernel, x, yerr, **kw)
    ranks = _level_ranks(s)
    top = max(max(v) for v in ranks.values())
    record_property("level_ranks", str(sorted((k, sorted(v)) for k, v in ranks.items())))
    if name == "general2d_short":
        assert top > 256
    rng = np.random.default_rng(n)
    Z = rng.standard_normal((n, 8))
    Y = s.apply_symmetric_factor(s.apply_symmetric_factor(Z, transpose=True))
    KZ, kfro = _ktilde_apply(s, kernel, x, yerr, Z)
    kz_err = float(np.sqrt(np.sum((Y.astype(LD) - KZ) ** 2)) / (kfro * np.sqrt(np.sum(Z * Z))))
    record_property("kz_err", kz_err)
    assert kz_err <= KZ_TOL
    per_level = {}
    for d in _internal(s):
        per_level[d["depth"]] = per_level.get(d["depth"], 0) + (d["rank"] > 0)
    expect_all = [per_level.get(l, 0) for l in range(len(per_level))]
    assert s.symmetric_factor_householder_nodes() == [0] * len(expect_all)  # every node took CholeskyQR3
    if n <= 1100:
        L, d = hiprec.ldlt_ld(_assemble(s, kernel, x, yerr))
        ref = np.sum(np.log(d))
        ld_err = float(abs(LD(s.symmetric_log_determinant) - ref) / abs(ref))
        record_property("logdet", ld_err)
        assert ld_err <= LDLT_TOL
    WZ = s.apply_symmetric_factor(Z)
    # the same factorisation with every node's bases from the Householder QR
    env.setenv("BGP_SYM_QR", "householder")
    s.compute(kernel, x, yerr, **kw)
    assert s.symmetric_factor_householder_nodes() == expect_all
    env.delenv("BGP_SYM_QR")
    WZh = s.apply_symmetric_factor(Z)
    Yh = s.apply_symmetric_factor(s.apply_symmetric_factor(Z, transpose=True))
    kz_err_h = float(np.sqrt(np.sum((Yh.astype(LD) - KZ) ** 2)) / (kfro * np.sqrt(np.sum(Z * Z))))
    record_property("kz_err_householder", kz_err_h)
    assert kz_err_h <= KZ_TOL
    qr_err = _relmax(WZh, WZ)
    record_property("qr_vs_householder", qr_err)
    assert qr_err <= QR_TOL


# ---- 7. apply widths and the C ABI ---------------------------------------------------------------------------------

def test_apply_widths_and_leading_dimension(gpu, env, record_property):
    from george_b200 import _lib
    from george_b200.solvers._hodlr import HODLRSolver
    kernel, ndim = _general("general2d")
    n = 1537
    x = _points(n, ndim)
    yerr = 0.1 * np.ones(n)
    s = HODLRSolver()
    s.compute(kernel, x, yerr, min_size=64, tol=1e-12, seed=42, rng_mode="pernode", exhaust="lowrank")
    W = s.apply_symmetric_factor(np.eye(n))
    Wt = s.apply_symmetric_factor(np.eye(n), transpose=True)
    lib = _lib.load()
    rng = np.random.default_rng(5)
    for nrhs in (1, 7, 8, 9, 63, 64, 65, 130):
        cols = rng.choice(n, nrhs, replace=False)
        Z = np.eye(n)[:, cols]
        # every column is its own sums, whatever the width and the group it falls in: bit for bit
        assert np.array_equal(s.apply_symmetric_factor(Z), W[:, cols]), nrhs
        assert np.array_equal(s.apply_symmetric_factor(Z, transpose=True), Wt[:, cols]), nrhs
        for transpose, ref in ((0, W), (1, Wt)):
            ld = n + 3
            B = np.full((ld, nrhs), -7.25, order="F")
            B[:n] = Z
            _lib.check(lib.bgp_hodlr_sym_apply(s._ptr, _lib.ptr(B), nrhs, ld, transpose))
            assert np.array_equal(B[:n], ref[:, cols]), (nrhs, transpose)
            assert np.all(B[n:] == -7.25), (nrhs, transpose)  # the padding rows are not touched


# ---- 8. wide levels ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [65536, 131072])
def test_wide_levels(gpu, env, record_property, n):
    """min_size = 1: the deepest internal level has n / 4 nodes of 2 or 3 rows (32768 and 65536 here), past a single
    launch's gridDim.y for the level products of compute(), the solves and the symmetric factor."""
    s, ou = _ou_solver(n, 1, "lowrank")
    internal = _internal(s)
    assert {d["rank"] for d in internal} == {1}
    width = {}
    for d in internal:
        width[d["depth"]] = width.get(d["depth"], 0) + 1
    record_property("widest_level", max(width.values()))
    assert max(width.values()) >= n // 4
    ref = ou.logdet()
    ld_err = float(abs(LD(s.log_determinant) - ref) / abs(ref))
    record_property("solver_logdet", ld_err)
    assert ld_err <= LOGDET_TOL
    B = np.random.default_rng(2).standard_normal((n, 3))
    X = s.apply_inverse(B)
    Xr = ou.solve(B)
    solve_err = float(np.sqrt(np.sum((X.astype(LD) - Xr) ** 2) / np.sum(Xr ** 2)))
    record_property("solve_err", solve_err)
    assert solve_err <= SOLVE_TOL
    _check_ou(s, ou, record_property, seed=n)
