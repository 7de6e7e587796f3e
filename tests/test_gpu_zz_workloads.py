# -*- coding: utf-8 -*-
"""bench.py's ExpSquared (cfg2) and quasi-periodic (cfg5) HODLR workloads at the sizes one GPU runs, against golden
vectors of the CPU oracle in the device's mode (per-node RNG streams, exhausted blocks keep their low-rank factors;
tests/golden/make_golden_workloads.py).

* cfg2: 1.0 * ExpSquared(1.0), N = 65536.
* cfg5: 1.0 * ExpSquared(1.0) + 0.5 * ExpSine2(1.0, log 3), N = 131072 (one GPU's share of bench.py's weak scaling).
  The periodic term never decays, so the ranks are large (a level of rank 382: the blocked partial-pivoting LU and the
  DMMA Gram slices of launch_level_big run on real data), and the shape has no decay bound (no candidate entry of the
  ACA is culled).

Unsharded, each golden: log-determinant, y^T K^-1 y and log-likelihood; a sample of K^-1 [y, b] (every 64th row, the
rows on both sides of every boundary of eight shards, the first and last rows); dot_solve against y . apply_inverse(y);
the tree geometry exactly; (rank, draws, fallback) on most internal nodes and the first min(2, rank) pivots of every
internal node (the rules of test_gpu_zz_fullsize.py: the last pivots at tol 1e-10 sit at the 1e-14 threshold).

Sharded: cfg5 at N = 131072 in eight host-exchange shards of 16384 rows on one device (test_gpu_hodlr_shards.py): every
node a shard factors has the unsharded handle's structure and pivots exactly, the partial log-determinants add up to
the unsharded one and the golden, and the split solve of [y, b] matches the unsharded handle and the golden sample,
shard boundaries included.  bench.py's eight-GPU size, N = 2^20, does not fit one 80 GB device: the unsharded
factorisation asks for one device buffer of 61.6 GB and fails, and each of eight shards would hold the top levels'
panels over all N rows.

Reference mode: rng_mode="reference", exhaust="dense" at bench.py's refmode_n (cfg2 16384, cfg5 8192) against the oracle
in the same mode, computed here (under a second of one core each): the assertion behind bench.py's
parity_reference_mode line.

Each case skips, saying what it found, when the free device memory is short of its measured need plus 4 GiB.  Errors,
wall time and the device memory held are recorded with ``record_property``.
"""
import os
import time

import numpy as np
import pytest

import test_gpu_hodlr_shards as sh
from test_gpu_zz_large_index import GB, _Memory, _release

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MIN_SIZE, TOL, SEED = 100, 1e-10, 42
SMALL_RANK_LIMIT = 142   # 2r above it: the blocked LU and the DMMA Gram slices (csrc/hodlr.cu: launch_level_big)

# Bars: 10-100x the largest error measured on one H100 80GB HBM3 (SXM, 700 W power limit) over three runs, scalars
# capped at 1e-9.  Where the cap cannot be met, the golden itself is not determined more closely: at tol = 1e-10 the
# last pivots of a node are residual entries at the 1e-14 rejection threshold, so which rows a node keeps depends on the
# last bit of its arithmetic.  The oracle compiled with fused multiply-adds (g++ -march=haswell -ffp-contract=fast), an
# equally exact restatement, differs from the golden by as much as the device does: cfg2 log-det 2.4e-13, quad 5.2e-11,
# solve 2.8e-7 and 501 of 511 nodes alike; cfg5 log-det 1.3e-10, quad 8.8e-8, log-likelihood 5.2e-8, solve 4.3e-4 and
# 902 of 1023 nodes alike.  K^-1 amplifies those choices by cond(K), which the periodic term makes large; the
# log-determinant, a sum over every node, is held below the cap in both workloads.
BARS = {
    "cfg2": dict(
        logdet=2e-11,   # |logdet - golden| / |golden|                                    (measured 4.2e-13)
        quad=1e-9,      # |y^T K^-1 y - golden| / |golden|                                (measured 1.4e-11)
        ll=5e-10,       # |log-likelihood - golden| / |golden|                            (measured 7.6e-12)
        solve=3e-6,     # max |X[rows] - golden| / max |golden|, worse of the columns      (measured 2.7e-7)
        dot=5e-14,      # |dot_solve(y) - y . apply_inverse(y)| / |.|                      (measured 6.6e-16)
        agree=0.9),     # share of internal nodes with the golden's (rank, draws, fallback) (measured 499 / 511)
    "cfg5": dict(
        logdet=1e-9,    #                                                                 (measured 1.6e-11)
        quad=1e-6,      #                                                                 (measured 7.0e-8)
        ll=5e-7,        #                                                                 (measured 4.1e-8)
        solve=5e-3,     #                                                                 (measured 4.3e-4)
        dot=1e-12,      #                                                                 (measured 2.5e-14)
        agree=0.8),     #                                                                 (measured 877 / 1023)
}
# Two runs of the same factorisation, and the eight shards against the unsharded handle, on the same device.  The Gram
# products of the big-rank levels add 4096-row slices with atomics, so two runs agree to rounding, not bits, and K^-1
# amplifies that rounding by cond(K) as it does in the golden comparison: the shards are as far from the unsharded
# handle as two unsharded runs are from each other (test_gpu_hodlr_shards.py measured 1.4e-13 on its
# better-conditioned problems).
REPEAT_BARS = dict(
    logdet=1e-11,     # |logdet - first run| / |first run|                                    (measured 4.8e-13)
    solve=1e-8,       # ||X - X_first run|| / ||X_first run||                                 (measured 6.9e-10)
)
SHARD_BARS = dict(
    logdet=1e-11,     # |sum of the 8 partial log-dets - unsharded| / |unsharded|            (measured 2.4e-13)
    solve=1e-8,       # ||X_sharded - X_unsharded|| / ||X_unsharded||                          (measured 8.1e-10)
    spread=1e-9,      # the eight shards' solves against shard 0's                             (measured 9.7e-11)
)
# The reference's own mode against the oracle: one shared stream, so the first node that keeps a different row changes
# the rows every later node draws (ranks of 83 of 127 and 19 of 63 internal nodes agree); the log-likelihood is
# compared (measured 3.2e-11 and 8.6e-9; the plain and the fused-multiply-add oracle are 1.9e-12 and 7.4e-8 apart).
REFMODE_LL = {"cfg2": 1e-9, "cfg5": 1e-7}
# device memory each case holds (the unsharded cfg5 case two handles at once), measured on the H100, bytes
NEED = {"cfg2_fullsize_n65536": 0.81e9, "cfg5_fullsize_n131072": 6.38e9}
SHARD_NEED = 15.6e9


def _kernel(workload):
    from george_b200 import kernels
    if workload == "cfg2":
        return 1.0 * kernels.ExpSquaredKernel(1.0)
    return 1.0 * kernels.ExpSquaredKernel(1.0) + 0.5 * kernels.ExpSine2Kernel(gamma=1.0, log_period=np.log(3.0))


def _data(n):
    """bench.py's inputs and the goldens' second right-hand side b = cos(0.37 x)."""
    rng = np.random.default_rng(1234)
    x = np.sort(rng.uniform(0, 10 * n / 1000, n))
    yerr = 0.1 * np.ones(n)
    y = np.sin(x) + 0.1 * rng.normal(size=n)
    return x, yerr, y, np.cos(0.37 * x)


def _golden(name):
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    assert int(g["n"]) == int(name.rsplit("_n", 1)[1])
    return g


def _tree(n, min_size):
    """(start, size, half, is_leaf, parent, direction, depth) of every node in pre-order: the reference's tree
    (hodlr.h:48-61: half = size // 2, a node splits iff half >= min_size)."""
    out = []

    def walk(start, size, parent, direction, depth):
        half = size // 2
        leaf = half < min_size
        i = len(out)
        out.append((start, size, half, int(leaf), parent, direction, depth))
        if not leaf:
            walk(start, half, i, 0, depth + 1)
            walk(start + half, size - half, i, 1, depth + 1)
    walk(0, n, -1, 0, 0)
    return out


GEOMETRY = ("start", "size", "half", "is_leaf", "parent", "direction", "depth")


def _check_nodes(s, g, n):
    """Geometry exactly and the first min(2, rank) pivots of every internal node.  Returns (internal nodes with the
    golden's (rank, draws, fallback), internal nodes)."""
    nodes = s.nodes()
    assert [tuple(nd[k] for k in GEOMETRY) for nd in nodes] == _tree(n, MIN_SIZE)
    assert [nd["is_leaf"] for nd in nodes] == g["is_leaf"].tolist()
    info, off, pr, pc = g["node_info"], g["piv_off"], g["piv_rows"], g["piv_cols"]
    inner = [i for i, nd in enumerate(nodes) if not nd["is_leaf"]]
    same = sum(1 for i in inner
               if (nodes[i]["rank"], nodes[i]["rng_draws"], nodes[i]["dense_fallback"]) == tuple(info[i].tolist()))
    for i in inner:
        k = min(2, nodes[i]["rank"], int(info[i, 0]))
        r, c = s.pivots(i, nodes[i]["rank"])
        assert r[:k].tolist() == pr[off[i]:off[i] + k].tolist() and c[:k].tolist() == pc[off[i]:off[i] + k].tolist(), i
    return same, len(inner)


def _sample_err(X, g):
    """Worse of the two columns of max |X[rows] - golden| / max |golden|."""
    rows = g["sample_rows"]
    return max(float(np.max(np.abs(X[rows, j] - g[key])) / np.max(np.abs(g[key])))
               for j, key in enumerate(("sample_y", "sample_b")))


def _level_ranks(nodes):
    """Largest rank per depth."""
    out = {}
    for nd in nodes:
        if not nd["is_leaf"]:
            out[nd["depth"]] = max(out.get(nd["depth"], 0), nd["rank"])
    return out


def _record(record_property, errs, mem):
    record_property("wall_s", round(time.time() - mem.t0, 1))
    record_property("device_gb_held", round(mem.held / GB, 2))
    for k, v in mem.stages.items():
        record_property("s:" + k, round(v, 2))
    for k, v in errs.items():
        record_property(k, "{0:.3g}".format(v))


def _compute(workload, x, yerr):
    from george_b200.solvers._hodlr import HODLRSolver
    s = HODLRSolver()
    s.compute(_kernel(workload), x[:, None], yerr, min_size=MIN_SIZE, tol=TOL, seed=SEED, rng_mode="pernode",
              exhaust="lowrank")
    return s


@pytest.fixture
def env(monkeypatch):
    for var in ("BGP_SMALL_RANK_LIMIT", "BGP_LEAF_COLS", "BGP_NO_GRAPH", "BGP_NO_CULL", "BGP_LEAF_FACTOR",
                "BGP_EVAL_MINB"):
        monkeypatch.delenv(var, raising=False)
    _release()
    yield monkeypatch
    _release()


CASES = ["cfg2_fullsize_n65536", "cfg5_fullsize_n131072"]


@pytest.mark.parametrize("name", CASES)
def test_unsharded_against_oracle_golden(gpu, env, record_property, name):
    mem = _Memory(NEED[name])
    g = _golden(name)
    workload, n = name.split("_")[0], int(g["n"])
    bars = BARS[workload]
    x, yerr, y, b = _data(n)
    s = _compute(workload, x, yerr)
    mem.check("compute")
    ld, quad = s.log_determinant, s.dot_solve(y)
    ll = -0.5 * (n * np.log(2 * np.pi) + ld) - 0.5 * quad
    X = s.apply_inverse(np.stack([y, b], axis=1))
    mem.check("solve")
    errs = dict(logdet=abs(ld - g["log_determinant"]) / abs(g["log_determinant"]),
                quad=abs(quad - g["quad"]) / abs(g["quad"]),
                ll=abs(ll - g["log_likelihood"]) / abs(g["log_likelihood"]),
                solve=_sample_err(X, g),
                dot=abs(quad - y @ X[:, 0]) / abs(y @ X[:, 0]))
    same, inner = _check_nodes(s, g, n)
    ranks = _level_ranks(s.nodes())
    prof, units = s.aca_profile(), s.eval_units()
    counts = {k: int(prof[k]) for k in ("evals", "evaluated", "candidates")}
    record_property("structure_agree", "{0}/{1}".format(same, inner))
    record_property("level_max_ranks", ranks)
    record_property("aca_counts", counts)
    record_property("eval_units", units)
    if workload == "cfg5":
        # the periodic sum has no decay bound: the same compute with culling switched off does the same work
        env.setenv("BGP_NO_CULL", "1")
        s2 = _compute(workload, x, yerr)
        env.delenv("BGP_NO_CULL")
        prof2 = s2.aca_profile()
        no_cull = ({k: int(prof2[k]) for k in counts}, s2.eval_units())
        # the Gram products add their row slices with atomics, so a repeat agrees to rounding, not bits
        errs["repeat_logdet"] = abs(s2.log_determinant - ld) / abs(ld)
        errs["repeat_solve"] = sh._rel(s2.apply_inverse(np.stack([y, b], axis=1)), X)
        mem.check("no_cull")
        del s2
    _record(record_property, errs, mem)
    bad = {k: (v, bars[k]) for k, v in errs.items() if k in bars and not v <= bars[k]}
    bad.update({k: (v, REPEAT_BARS[k[7:]]) for k, v in errs.items()
                if k.startswith("repeat_") and not v <= REPEAT_BARS[k[7:]]})
    assert not bad, bad
    assert same >= bars["agree"] * inner, (same, inner)
    if workload == "cfg5":
        assert max(2 * r for r in ranks.values()) > SMALL_RANK_LIMIT, ranks
        assert no_cull == (counts, units), (no_cull, counts, units)
        # every verified entry was evaluated; a2_eval also evaluates the speculative candidates past each winner, so
        # "evaluated" exceeds "evals" here
        assert counts["evaluated"] >= counts["evals"], counts


def test_cfg5_in_eight_shards(gpu, env, record_property):
    """cfg5 at N = 131072 in eight host-exchange shards on one device."""
    from george_b200.solvers._hodlr import HODLRSolver
    mem = _Memory(SHARD_NEED)
    P = 8
    g = _golden("cfg5_fullsize_n131072")
    n = int(g["n"])
    x, yerr, y, b = _data(n)
    kernel = _kernel("cfg5")
    opts = dict(min_size=MIN_SIZE, tol=TOL, exhaust="lowrank")
    single = sh._single(kernel, x[:, None], yerr, **opts)
    mem.check("single")
    B = np.stack([y, b], axis=1)
    X1 = single.apply_inverse(B)
    ld1 = single.log_determinant
    del single
    # the unsharded factorisation once more: how far two runs of the same path are apart
    single = sh._single(kernel, x[:, None], yerr, **opts)
    repeat = dict(repeat_logdet=abs(single.log_determinant - ld1) / abs(ld1),
                  repeat_solve=sh._rel(single.apply_inverse(B), X1))
    shards = sh._shards(kernel, x[:, None], yerr, P, **opts)
    mem.check("shards")
    compared = sh._check_structure(shards, single, n, MIN_SIZE)
    outs = sh._sharded_solve(shards, B)
    mem.check("solve")
    errs = dict(logdet=abs(shards.log_determinant - ld1) / abs(ld1),
                logdet_golden=abs(shards.log_determinant - g["log_determinant"]) / abs(g["log_determinant"]),
                solve=sh._rel(outs[0], X1),
                spread=max(sh._rel(o, outs[0]) for o in outs[1:]),
                solve_golden=_sample_err(outs[0], g), **repeat)
    record_property("nodes_compared", compared)
    _record(record_property, errs, mem)
    del single, shards
    HODLRSolver.release_parked()
    assert errs["logdet"] <= SHARD_BARS["logdet"] and errs["logdet_golden"] <= BARS["cfg5"]["logdet"], errs
    assert errs["solve"] <= SHARD_BARS["solve"] and errs["spread"] <= SHARD_BARS["spread"], errs
    assert errs["repeat_logdet"] <= REPEAT_BARS["logdet"] and errs["repeat_solve"] <= REPEAT_BARS["solve"], errs
    assert errs["solve_golden"] <= BARS["cfg5"]["solve"], errs


@pytest.mark.parametrize("workload,n", [("cfg2", 16384), ("cfg5", 8192)])
def test_reference_mode_parity(gpu, env, oracle, record_property, workload, n):
    """bench.py's parity_reference_mode: one shared mt19937 and exhausted blocks stored densely, against the oracle in
    the same mode."""
    from george_b200._spec import flatten
    from george_b200.solvers._hodlr import HODLRSolver
    x, yerr, y, _ = _data(n)
    kernel = _kernel(workload)
    t0 = time.time()
    o = oracle.HODLR(flatten(kernel), x, yerr, min_size=MIN_SIZE, tol=TOL, seed=SEED, rng_mode=1, exhaust=0)
    ll_ref = -0.5 * (n * np.log(2 * np.pi) + o.log_determinant) - 0.5 * o.dot_solve(y)
    record_property("oracle_s", round(time.time() - t0, 2))
    s = HODLRSolver()
    s.compute(kernel, x[:, None], yerr, min_size=MIN_SIZE, tol=TOL, seed=SEED, rng_mode="reference", exhaust="dense")
    ll = -0.5 * (n * np.log(2 * np.pi) + s.log_determinant) - 0.5 * s.dot_solve(y)
    err = abs(ll - ll_ref) / abs(ll_ref)
    got, want = s.nodes(), o.nodes()
    inner = [i for i, nd in enumerate(want) if not nd["is_leaf"]]
    record_property("ll", "{0:.3g}".format(err))
    record_property("ranks_agree", "{0}/{1}".format(sum(1 for i in inner if got[i]["rank"] == want[i]["rank"]),
                                                    len(inner)))
    assert [tuple(nd[k] for k in GEOMETRY) for nd in got] == [tuple(nd[k] for k in GEOMETRY) for nd in want]
    # the root draws first from the seeded stream
    assert (got[0]["rank"], got[0]["rng_draws"]) == (want[0]["rank"], want[0]["rng_draws"])
    assert [nd["dense_fallback"] for nd in got] == [nd["dense_fallback"] for nd in want]
    assert err <= REFMODE_LL[workload], err
