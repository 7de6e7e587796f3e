# -*- coding: utf-8 -*-
"""Which candidate-evaluation work the lock-step ACA publishes (csrc/hodlr_aca2.cuh: a2_generate / a2_eval_kernel).

a2_generate publishes an eval item (column chunk, block of live candidates) only when a bound over the whole chunk and
the whole block cannot rule out every (candidate, 128-column group) pair of it; a2_eval then bounds each pair again and
evaluates the survivors.  Dropping an item must never drop a pair a2_eval would have evaluated, so everything the ACA
decides and counts is what the build that published every chunk produced.  The constants below were recorded with
that build (one H100 80GB HBM3) on the same inputs: the verified, evaluated and update counts, the candidates, the
lock-step iterations, the rare draw paths, the per-node ranks and the pivot lists (as a SHA-256 of the int64 rows and
columns, node by node in pre-order).  The units that build pulled (one unit = one item against one 128-column group) are
recorded too: with a decaying kernel fewer are pulled now, and with the periodic sum, which has no bound, exactly as
many.
"""
import hashlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_FULL = 65536


def _kernel(name):
    from george_b200 import kernels as K
    if name == "m32":        # the headline's kernel and leaf size
        return 1.0 * K.Matern32Kernel(1.0), 256
    if name == "expsq":
        return 1.0 * K.ExpSquaredKernel(1.0), 100
    # the config-5 sum: a periodic term never decays, so nothing is culled and every chunk is published
    return 1.0 * K.ExpSquaredKernel(1.0) + 0.5 * K.ExpSine2Kernel(gamma=1.0, log_period=np.log(3.0)), 100


def _data(n):
    """bench.py's synthetic inputs: n sorted uniform coordinates on [0, n / 100), unit noise 0.1."""
    rng = np.random.default_rng(1234)
    x = np.sort(rng.uniform(0, 10 * n / 1000, n))
    return x, 0.1 * np.ones(n)


def _digest(arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a, dtype=np.int64).tobytes())
    return h.hexdigest()


def observe(s):
    """What the last compute of native solver `s` decided and counted."""
    nodes = s.nodes()
    internal = [i for i, nd in enumerate(nodes) if not nd["is_leaf"]]
    ranks = [nodes[i]["rank"] for i in internal]
    piv = []
    for i in internal:
        r, c = s.pivots(i, nodes[i]["rank"])
        piv += [r, c]
    prof = s.aca_profile()
    return {"counts": {k: int(prof[k]) for k in ("evals", "candidates", "evaluated", "update_fmas", "eval_launches")},
            "draw_paths": s.draw_paths(), "rank_sum": int(sum(ranks)), "ranks": _digest([ranks]),
            "pivots": _digest(piv), "units": s.eval_units()}


def compute(name, n=N_FULL):
    from george_b200.solvers._hodlr import HODLRSolver
    kernel, min_size = _kernel(name)
    x, yerr = _data(n)
    s = HODLRSolver()
    s.compute(kernel, x[:, None], yerr, min_size=min_size, tol=1e-10, seed=42, rng_mode="pernode", exhaust="lowrank")
    return s


RECORDED = {'m32': {'counts': {'evals': 340664576,
                    'candidates': 91721,
                    'evaluated': 55239040,
                    'update_fmas': 108680832,
                    'eval_launches': 10},
         'draw_paths': {'lemire_redos': 0, 'truncated_batches': 0, 'sequential_draws': 0, 'partial_commits': 350},
         'rank_sum': 603,
         'ranks': '0eb6652fa2dce8e9bece25e7ef07d2f3d9d8c605354cb14ffd5915bd44085f87',
         'pivots': 'e28936e345a447545626ce3022eed3e7913816153d712ec09b4c48a95cdfbbb7',
         'units_pulled': 113840},
 'expsq': {'counts': {'evals': 129874688,
                      'candidates': 17365,
                      'evaluated': 10663552,
                      'update_fmas': 117291264,
                      'eval_launches': 36},
           'draw_paths': {'lemire_redos': 0,
                          'truncated_batches': 0,
                          'sequential_draws': 0,
                          'partial_commits': 1654},
           'rank_sum': 6028,
           'ranks': '121887e6e8bbee6f3f3e2e2b8aa53c6820a225ff9117f9c3e2996d1e2b233329',
           'pivots': '140a398f7e66b2b55fa0d33a2bd35e4bcc98a82e824aeec0526c81a96828da83',
           'units_pulled': 87576},
 'sum_expsq_es2': {'counts': {'evals': 38333824,
                              'candidates': 14861,
                              'evaluated': 65566208,
                              'update_fmas': 3790365696,
                              'eval_launches': 815},
                   'draw_paths': {'lemire_redos': 0,
                                  'truncated_batches': 0,
                                  'sequential_draws': 0,
                                  'partial_commits': 1366},
                   'rank_sum': 12310,
                   'ranks': '09a9443b8c53979d1a6b5e55b048385a4e43c146587220612ae8a9d5bd3becce',
                   'pivots': 'fb33e847fce0aea2bb1394e95ce33ff837feb33d020406c9608ab9a809a7b499',
                   'units_pulled': 82152}}


@pytest.fixture
def clean_env(monkeypatch):
    for var in ("BGP_NO_GRAPH", "BGP_NO_CULL", "BGP_EVAL_MINB"):
        monkeypatch.delenv(var, raising=False)
    return monkeypatch


@pytest.mark.parametrize("name", ["m32", "expsq", "sum_expsq_es2"])
def test_decisions_and_counts_match_the_build_that_published_every_chunk(gpu, clean_env, record_property, name):
    got = observe(compute(name))
    want = RECORDED[name]
    record_property("units", got["units"])
    for key in ("counts", "draw_paths", "rank_sum", "ranks", "pivots"):
        assert got[key] == want[key], (key, got[key], want[key])
    assert 0 < got["units"]["live"] <= got["units"]["pulled"]
    if name == "sum_expsq_es2":  # no bound: every chunk is published
        assert got["units"]["pulled"] == want["units_pulled"]
    else:
        assert got["units"]["pulled"] < want["units_pulled"]


def _edge_groups_problem():
    """Root of 4096 points: the right half's rows sit in [100, 120]; of the left half's columns only the first and the last
    128-column group of chunk 0 lie next to them ([95, 100)), the six groups between and all of chunk 1 lie 50 and more
    length scales away.  Every live pair of the root is in the two edge groups of one chunk."""
    rng = np.random.default_rng(7)
    n = 4096
    x = np.empty(n)
    near = np.r_[0:128, 896:1024]
    far = np.setdiff1d(np.arange(2048), near)
    x[near] = 95.0 + 5.0 * rng.random(near.size)
    x[far] = 50.0 * rng.random(far.size)
    x[2048:] = np.sort(100.0 + 20.0 * rng.random(2048))
    return x


@pytest.mark.parametrize("kname", ["m32", "expsq"])
def test_live_pairs_only_in_the_edge_groups_of_a_chunk(gpu, clean_env, kname):
    """The chunk's range is the union of its groups' ranges: an item whose live pairs sit only in the chunk's first and
    last group is kept, and everything is decided as by the exhaustive scan (BGP_NO_CULL)."""
    from george_b200 import kernels as K
    from george_b200.solvers._hodlr import HODLRSolver
    kernel = {"m32": 1.0 * K.Matern32Kernel(1.0), "expsq": 1.0 * K.ExpSquaredKernel(1.0)}[kname]
    x = _edge_groups_problem()
    yerr = 0.1 * np.ones(x.size)
    y = np.sin(x)
    res = {}
    for cull in (True, False):
        if cull:
            clean_env.delenv("BGP_NO_CULL", raising=False)
        else:
            clean_env.setenv("BGP_NO_CULL", "1")
        s = HODLRSolver()
        s.compute(kernel, x[:, None], yerr, min_size=256, tol=1e-10, seed=42, rng_mode="pernode", exhaust="lowrank")
        res[cull] = (observe(s), s.log_determinant, s.dot_solve(y))
    clean_env.delenv("BGP_NO_CULL", raising=False)
    on, off = res[True][0], res[False][0]
    for key in ("draw_paths", "rank_sum", "ranks", "pivots"):
        assert on[key] == off[key], (key, on[key], off[key])
    for key in ("evals", "candidates", "eval_launches"):
        assert on["counts"][key] == off["counts"][key], key
    assert on["counts"]["evaluated"] <= off["counts"]["evaluated"]
    assert abs(res[True][1] - res[False][1]) <= 1e-13 * abs(res[False][1])
    assert abs(res[True][2] - res[False][2]) <= 1e-12 * abs(res[False][2])
    # the far chunk's items were not published; the root's edge groups were evaluated
    assert 0 < on["units"]["live"] <= on["units"]["pulled"] < off["units"]["pulled"]
