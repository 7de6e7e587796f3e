# -*- coding: utf-8 -*-
"""The dense building blocks of the big-rank Woodbury step (csrc/hodlr_lu.cuh, csrc/gemm_dmma.cuh) against LAPACK,
and the HODLR solver on cases whose ranks take that path (2r > 142) against the oracle."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


GD_ATOMIC_ADD, GD_LOWER = 1, 256


def _gemm(lib, a_k, b_k, A, B, Cm, mode):
    """A, B: stored arrays (column-major semantics handled by the caller), returns updated C (m x n)."""
    from george_b200 import _lib
    m, n = Cm.shape
    k = A.shape[1] if a_k == 0 else A.shape[0]
    # column-major storage = Fortran order
    Af = np.asfortranarray(A)
    Bf = np.asfortranarray(B)
    Cf = np.asfortranarray(Cm.copy())
    _lib.check(lib.bgp_selftest_gemm(a_k, b_k, m, n, k, _lib.ptr(Af), Af.shape[0], _lib.ptr(Bf), Bf.shape[0],
                                     _lib.ptr(Cf), Cf.shape[0], mode))
    return Cf


@pytest.mark.parametrize("m,n,k", [(1, 1, 1), (128, 128, 16), (200, 150, 70), (1000, 1, 32), (37, 300, 4100),
                                   (513, 129, 33)])
@pytest.mark.parametrize("a_k", [0, 1])
def test_dmma_gemm_variants(gpu, m, n, k, a_k):
    """Every (a_kcontig, b_kcontig) variant in the subtracting, atomic-adding and lower-only modes; the lower-only
    mode leaves the entries above the diagonal untouched."""
    from george_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(m * 7 + n * 3 + k)
    Ap = rng.normal(size=(m, k))          # A' (m x k)
    Bp = rng.normal(size=(k, n))          # B' (k x n)
    C0 = rng.normal(size=(m, n))
    A_store = Ap if a_k == 0 else Ap.T.copy()   # a_k=0: M x K column-major; a_k=1: K x M column-major
    lower = np.tril(np.ones((m, n), dtype=bool))
    for b_k in (0, 1):
        B_store = Bp if b_k == 1 else Bp.T.copy()  # b_k=1: K x N column-major; b_k=0: N x K column-major
        for mode in (0, GD_ATOMIC_ADD, GD_LOWER):
            got = _gemm(lib, a_k, b_k, A_store, B_store, C0, mode)
            want = C0 + Ap @ Bp if mode == GD_ATOMIC_ADD else C0 - Ap @ Bp
            if mode == GD_LOWER:
                assert np.array_equal(got[~lower], C0[~lower]), (b_k, mode)
                got, want = got[lower], want[lower]
            np.testing.assert_allclose(got, want, rtol=0, atol=1e-11 * max(1.0, np.sqrt(k)), err_msg=str((b_k, mode)))


@pytest.mark.parametrize("n,e,b,cend", [
    (2100, 64, 0, 256),      # rank-64 update inside the first MB block
    (2100, 256, 0, 2048),    # rank-MB update up to the OB boundary
    (2100, 2048, 0, 2100),   # rank-OB update, ragged 52-row remainder
    (4161, 2048, 0, 4161),   # rank-OB update of a 2113-row trailing matrix
    (4161, 4096, 2048, 4161),  # second OB block, 65-row remainder
    (700, 640, 512, 700),    # rank-128 update of a 60-row tail (small-OB blocking)
    (577, 576, 512, 577),    # last panel of width 1
    (129, 64, 0, 128)])      # one row below the update's columns
def test_dmma_gemm_cholesky_update(gpu, n, e, b, cend):
    """The <A M-contiguous, B N-contiguous> variant with the lower-only output: exactly the descriptors dense_potrf
    issues, C[e:n, e:cend) -= L[e:n, b:e) L[e:cend, b:e)^T with A and B the same panel.  Entries above the diagonal
    are left untouched, in the lower-only and in the full mode."""
    from george_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(n + e + cend)
    M, N, K = n - e, cend - e, e - b
    P = np.asfortranarray(rng.normal(size=(M, K)))  # rows e.., columns b..e of the factor (leading dimension M)
    C0 = np.asfortranarray(rng.normal(size=(M, N)))
    full = C0 - P @ P[:N].T
    lower = np.tril(np.ones((M, N), dtype=bool))
    for mode in (0, GD_LOWER):
        Cf = C0.copy(order="F")
        _lib.check(lib.bgp_selftest_gemm(0, 0, M, N, K, _lib.ptr(P), M, _lib.ptr(P), M, _lib.ptr(Cf), M, mode))
        if mode == GD_LOWER:
            assert np.array_equal(Cf[~lower], C0[~lower])
            np.testing.assert_allclose(Cf[lower], full[lower], rtol=0, atol=1e-11 * np.sqrt(K))
        else:
            np.testing.assert_allclose(Cf, full, rtol=0, atol=1e-11 * np.sqrt(K))


@pytest.mark.parametrize("n,nrhs", [(1, 1), (31, 3), (32, 1), (33, 5), (64, 64), (150, 1), (257, 200), (700, 130)])
def test_blocked_lu_vs_lapack(gpu, n, nrhs):
    from george_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(n + nrhs)
    if n >= 2 and n % 2 == 0:
        r = n // 2  # the Woodbury shape [[I, A], [B, I]]
        S = np.eye(n)
        S[:r, r:] = rng.normal(size=(r, r)) / np.sqrt(r)
        S[r:, :r] = rng.normal(size=(r, r)) / np.sqrt(r)
    else:
        S = rng.normal(size=(n, n)) + 0.5 * np.eye(n)
    R = rng.normal(size=(n, nrhs))
    Sf = np.asfortranarray(S)
    Rf = np.asfortranarray(R.copy())
    ld = C.c_double(0.0)
    _lib.check(lib.bgp_selftest_lu(n, nrhs, _lib.ptr(Sf), _lib.ptr(Rf), C.byref(ld)))
    want = np.linalg.solve(S, R)
    cond = np.linalg.cond(S)
    assert np.linalg.norm(Rf - want) <= 1e-13 * cond * np.linalg.norm(want) + 1e-14
    assert abs(ld.value - np.linalg.slogdet(S)[1]) <= 1e-11 * max(1.0, abs(ld.value)) * max(1.0, np.log10(cond))


@pytest.mark.parametrize("n,col", [(144, 5), (162, 161)])
def test_blocked_lu_with_a_nan_column_returns_nan(gpu, n, col):
    """A Woodbury matrix whose trailing column is NaN below the diagonal (what non-finite kernel values or noise produce)
    has no comparable pivot candidate there.  The panel kernel keeps the row in place and the NaN reaches log|det| and
    the solve, as the shared-memory path does; it used to take the arg-max's 'nothing found' sentinel as a row index.
    The handle stays usable afterwards."""
    from george_b200 import _lib
    lib = _lib.load()
    S = np.eye(n)
    S[col:, col] = np.nan
    Sf = np.asfortranarray(S)
    Rf = np.asfortranarray(np.ones((n, 3)))
    ld = C.c_double(0.0)
    _lib.check(lib.bgp_selftest_lu(n, 3, _lib.ptr(Sf), _lib.ptr(Rf), C.byref(ld)))
    assert np.isnan(ld.value)
    assert np.all(np.isnan(Rf[col]))
    # the device is still healthy: a regular system right after
    S = np.eye(n) + 0.1 * np.random.default_rng(n).normal(size=(n, n)) / np.sqrt(n)
    Sf, Rf = np.asfortranarray(S), np.asfortranarray(np.ones((n, 1)))
    _lib.check(lib.bgp_selftest_lu(n, 1, _lib.ptr(Sf), _lib.ptr(Rf), C.byref(ld)))
    np.testing.assert_allclose(Rf[:, 0], np.linalg.solve(S, np.ones(n)), rtol=0, atol=1e-12)


def test_big_rank_levels_match_oracle(gpu, oracle):
    """ExpSquared + ExpSine2 at N = 16384: the reference algorithm's ranks reach ~75 at the top (2r > 142), so the top
    levels take the blocked-LU / DMMA path and the lower ones the shared-memory path."""
    import bench
    from george_b200.solvers._hodlr import HODLRSolver
    from george_b200._spec import flatten
    n = 16384
    kernel = bench.make_kernel("cfg5")
    rng = np.random.default_rng(1234)
    x = np.sort(rng.uniform(0, 10 * n / 1000, n))[:, None]
    yerr = 0.1 * np.ones(n)
    y = np.sin(x[:, 0]) + 0.1 * rng.normal(size=n)
    o = oracle.HODLR(flatten(kernel), x, yerr, min_size=100, tol=1e-10, seed=42, rng_mode=0)
    s = HODLRSolver()
    s.compute(kernel, x, yerr, min_size=100, tol=1e-10, seed=42)
    gn, on = s.nodes(), o.nodes()
    assert max(nd["rank"] for nd in on) > 71 and max(nd["rank"] for nd in gn) > 71
    # the tail of this kernel's ACA runs at the rounding-noise floor (accepted pivots ~1e-13), so the last few ranks
    # depend on the last bits of exp/sin: same tree, ranks within a few of the oracle's, values to tolerance
    assert [nd["is_leaf"] for nd in gn] == [nd["is_leaf"] for nd in on]
    assert max(abs(a_["rank"] - b_["rank"]) for a_, b_ in zip(gn, on)) <= 8
    assert abs(s.log_determinant - o.log_determinant) <= 1e-9 * abs(o.log_determinant)
    assert abs(s.dot_solve(y) - o.dot_solve(y)) <= 1e-7 * abs(o.dot_solve(y))
    # K is ill-conditioned here (non-decaying periodic term: cond ~ 1e6) and the two factorisations differ in their
    # noise-floor ranks, so the solutions are compared through their residuals on a sample of rows: the device
    # solve must be as accurate as the reference algorithm's
    a, ao = s.apply_inverse(y)[:, 0], o.apply_inverse(y)
    rows = np.random.default_rng(7).choice(n, 256, replace=False)
    Kr = oracle.value_general(flatten(kernel), x[rows], x)
    res_g = np.linalg.norm(Kr @ a + yerr[rows] ** 2 * a[rows] - y[rows])
    res_o = np.linalg.norm(Kr @ ao + yerr[rows] ** 2 * ao[rows] - y[rows])
    assert res_g <= max(10.0 * res_o, 1e-8 * np.linalg.norm(y[rows]))
    assert np.linalg.norm(a - ao) <= 1e-4 * np.linalg.norm(ao)  # each is ~7e-6 from the dense solve (cond ~ 1e6)


@pytest.mark.parametrize("kname", ["expsq", "m52_3d"])
def test_every_level_through_the_big_path(gpu, oracle, monkeypatch, kname):
    """BGP_SMALL_RANK_LIMIT=0 sends all levels (any rank) through the DMMA Gram/update + blocked LU path; the result
    must agree with the shared-memory path and the oracle."""
    from george_b200 import kernels as K
    from george_b200.solvers._hodlr import HODLRSolver
    from george_b200._spec import flatten
    rng = np.random.default_rng(5)
    n = 3000
    if kname == "m52_3d":
        x = rng.uniform(0, 1, (n, 3))
        x = x[np.argsort(x[:, 0])]
        kernel, tol = 1.0 * K.Matern52Kernel(0.5, ndim=3), 1e-12
    else:
        x = np.sort(rng.uniform(0, 10 * n / 1000, n))[:, None]
        kernel, tol = 1.0 * K.ExpSquaredKernel(1.0), 1e-10
    yerr = 0.1 * np.ones(n)
    y = rng.normal(size=(n, 3))
    res = {}
    for limit in ("142", "0"):
        monkeypatch.setenv("BGP_SMALL_RANK_LIMIT", limit)
        s = HODLRSolver()
        s.compute(kernel, x, yerr, min_size=100, tol=tol, seed=42)
        res[limit] = (s.log_determinant, s.apply_inverse(y), s.dot_solve(y[:, 0]))
    o = oracle.HODLR(flatten(kernel), x, yerr, min_size=100, tol=tol, seed=42, rng_mode=0)
    for limit in res:
        assert abs(res[limit][0] - o.log_determinant) <= 1e-9 * abs(o.log_determinant)
        assert abs(res[limit][2] - o.dot_solve(y[:, 0])) <= 1e-7 * abs(o.dot_solve(y[:, 0]))
    assert np.linalg.norm(res["0"][1] - res["142"][1]) <= 1e-8 * np.linalg.norm(res["142"][1])
