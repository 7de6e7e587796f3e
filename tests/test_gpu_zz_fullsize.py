# -*- coding: utf-8 -*-
"""Size-independent properties at BASELINE.json's full sizes for the configurations the oracle cannot reach
(config 3 is covered by tests/test_gpu_ops.py::test_full_size_round_trip).

* config 2 (ExpSquared 1-D, N = 65536, HODLR tol = 1e-10): K (K^-1 y) == y with K applied matrix-free, to the
  north-star bar 1e-6; log-likelihood identical (1e-9) between the two RNG-independent ways of computing the quadratic
  form (dot_solve vs y . apply_inverse); two computes give the same log-det to 1e-12.
* config 4 (Matern52 3-D, N = 32768, dense Cholesky): the same round trip through the dense solver.

Configs 2 and 5 (bench.py's cfg2 and cfg5, N = 65536, 131072 and 2^20, unsharded and in eight shards) are held to
golden vectors of the CPU oracle at full size in tests/test_gpu_zz_workloads.py.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def test_config2_full_size_round_trip(gpu):
    import george_b200 as george
    from george_b200 import kernels
    n = 65536
    rng = np.random.default_rng(1234)
    x = np.sort(rng.uniform(0, 10 * n / 1000, n))
    yerr = 0.1 * np.ones(n)
    y = np.sin(x) + 0.1 * rng.normal(size=n)
    kernel = 1.0 * kernels.ExpSquaredKernel(1.0)
    s = george.HODLRSolver(kernel, tol=1e-10, seed=42, exhaust="lowrank")   # as bench.py --workload cfg2
    s.compute(x[:, None], yerr)
    ld = s.log_determinant
    assert np.isfinite(ld)
    b = s.apply_inverse(y)[:, 0]
    back = kernel.matvec(x[:, None], x[:, None], b, diag=yerr ** 2)
    assert np.linalg.norm(back - y) <= 1e-6 * np.linalg.norm(y)
    assert abs(s.dot_solve(y) - y @ b) <= 1e-9 * abs(y @ b)
    s2 = george.HODLRSolver(kernel, tol=1e-10, seed=42, exhaust="lowrank")
    s2.compute(x[:, None], yerr)
    assert abs(s2.log_determinant - ld) <= 1e-12 * abs(ld)  # split-K reductions use floating-point atomics


def test_config4_full_size_round_trip(gpu):
    import george_b200 as george
    from george_b200 import kernels
    n = 32768
    rng = np.random.default_rng(1234)
    x = rng.uniform(0, 1, (n, 3))
    x = x[np.argsort(x[:, 0])]
    yerr = 0.1 * np.ones(n)
    y = np.sin(x.sum(axis=1)) + 0.1 * rng.normal(size=n)
    kernel = 1.0 * kernels.Matern52Kernel(0.5, ndim=3)
    s = george.BasicSolver(kernel)
    s.compute(x, yerr)
    assert np.isfinite(s.log_determinant)
    b = s.apply_inverse(y)
    back = kernel.matvec(x, x, b, diag=yerr ** 2)
    assert np.linalg.norm(back - y) <= 1e-7 * np.linalg.norm(y)  # n = 8192 reaches 1e-9 (tests/test_gpu_dense.py)
    assert abs(s.dot_solve(y) - y @ b) <= 1e-9 * abs(y @ b)


@pytest.mark.parametrize("n", [65536, 262144])
def test_config3_full_size_against_oracle_golden(gpu, n):
    """BASELINE.json configs[2] (the headline: Matern32 1-D, N = 262144, leaf 256) against golden vectors produced by the
    CPU oracle in the SAME mode (per-node RNG streams, exhausted blocks keep their factors) at the FULL size
    (tests/golden/make_golden_fullsize.py: 512 s of one core at N = 262144).  Scalars to 1e-9 relative (north-star bar:
    1e-6).  Matern-3/2 is exactly rank 2 on sorted 1-D inputs, so whether a node finds a third, rounding-noise pivot
    (>= 1e-14) or exhausts its rows depends on the last bit of exp(): ranks and draw counts are compared node by node
    but only required to agree on >= 90 % of the nodes; the first two pivots of every node (the ones that carry the
    block) must be identical."""
    import os
    from george_b200 import kernels
    from george_b200.solvers._hodlr import HODLRSolver
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cfg3_fullsize_n{0}.npz".format(n))
    g = np.load(path)
    assert int(g["n"]) == n
    rng = np.random.default_rng(1234)
    x = np.sort(rng.uniform(0, 10 * n / 1000, n))
    yerr = 0.1 * np.ones(n)
    y = np.sin(x) + 0.1 * rng.normal(size=n)
    s = HODLRSolver()
    s.compute(1.0 * kernels.Matern32Kernel(1.0), x[:, None], yerr, min_size=256, tol=1e-10, seed=42, exhaust="lowrank")
    ld, quad = s.log_determinant, s.dot_solve(y)
    ll = -0.5 * (n * np.log(2 * np.pi) + ld) - 0.5 * quad
    assert abs(ld - float(g["log_determinant"])) <= 1e-9 * abs(float(g["log_determinant"]))
    assert abs(quad - float(g["quad"])) <= 1e-9 * abs(float(g["quad"]))
    assert abs(ll - float(g["log_likelihood"])) <= 1e-9 * abs(float(g["log_likelihood"]))
    nodes = s.nodes()
    info = g["node_info"]
    assert len(nodes) == len(info)
    assert [nd["is_leaf"] for nd in nodes] == [int(v) for v in info[:, 3]]
    inner = [i for i, nd in enumerate(nodes) if not nd["is_leaf"]]
    same = sum(1 for i in inner if (nodes[i]["rank"], nodes[i]["rng_draws"], nodes[i]["dense_fallback"]) == tuple(int(v) for v in info[i, :3]))
    assert same >= 0.9 * len(inner), (same, len(inner))
    off, pr, pc = g["piv_off"], g["piv_rows"], g["piv_cols"]
    for i in inner:
        k = min(2, nodes[i]["rank"], int(info[i, 0]))
        r, c = s.pivots(i, nodes[i]["rank"])
        assert list(r[:k]) == list(pr[off[i]:off[i] + k]) and list(c[:k]) == list(pc[off[i]:off[i] + k]), i


def test_small_and_big_woodbury_paths_agree_on_a_deep_tree(gpu, monkeypatch):
    """ExpSquared, N = 262144, leaves of 128: 2047 internal nodes on 11 levels, ranks 8..21, 205 factor columns.  Every level
    goes through the one-CTA-per-node Woodbury step (complete-pivoting LU in shared memory) by default and through the
    blocked LU + DMMA products when BGP_SMALL_RANK_LIMIT forces it; both must give the same log-determinant and solve
    (regression: a thread re-reading the pivot entry after a neighbour had started the row swap took the "singular"
    branch — NaN on ~3 % of the 1024 deepest nodes, only with many CTAs in flight)."""
    from george_b200 import kernels
    from george_b200.solvers._hodlr import HODLRSolver
    n = 262144
    rng = np.random.default_rng(1234)
    x = np.sort(rng.uniform(0, 10 * n / 1000, n))
    yerr = 0.1 * np.ones(n)
    y = np.sin(x) + 0.1 * rng.normal(size=n)
    res = {}
    for big in (False, True):
        if big:
            monkeypatch.setenv("BGP_SMALL_RANK_LIMIT", "1")
        else:
            monkeypatch.delenv("BGP_SMALL_RANK_LIMIT", raising=False)
        s = HODLRSolver()
        s.compute(1.0 * kernels.ExpSquaredKernel(1.0), x[:, None], yerr, min_size=100, tol=1e-10, seed=42, exhaust="lowrank")
        res[big] = (s.log_determinant, s.dot_solve(y))
    monkeypatch.delenv("BGP_SMALL_RANK_LIMIT", raising=False)
    assert np.isfinite(res[False][0]) and np.isfinite(res[False][1])
    assert abs(res[False][0] - res[True][0]) <= 1e-11 * abs(res[True][0])
    assert abs(res[False][1] - res[True][1]) <= 1e-9 * abs(res[True][1])
