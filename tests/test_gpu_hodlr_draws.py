# -*- coding: utf-8 -*-
"""The speculative row draws of the lock-step ACA (csrc/hodlr_aca2.cuh: a2_generate / a2_decide) against an independent
model of the reference's RNG loop (tests/aca_draw_model.py, pinned to libstdc++ by tests/test_aca_draw_model.py).

The device draws up to 8192 candidate rows at once, redoes Lemire rejections after the fact, resolves the swap-pop of
the row list through a multimap with writer chains and commits only the draws consumed.  None of that is visible on a
smooth kernel, where every row is usable or every row is rejected.  Here the blocks are partial permutation patterns
(``aca_draw_model.Problem``): a row is usable iff it was made special, so ranks, pivot rows and columns, the words
drawn and the exhaustion flag of every node are a pure function of the draw order, and the special rows are chosen
AFTER running the model so that a winner sits where a given path of the device code is taken.  The path counters of
``bgp_hodlr_last_draw_paths`` show that it was.  K_h is then known in closed form (1 x 1 and 2 x 2 blocks) and log-det,
solves and dot_solve are compared with it in longdouble.
"""

import numpy as np
import pytest

import aca_draw_model as M

pytestmark = pytest.mark.gpu

LD = np.longdouble
YERR = 0.1
# bars: 15-50x the largest value measured on one H100 80GB HBM3 (700 W power limit); cond(K_h) <= 8.6 (d = 1.01, |a| <= 0.8)
LOGDET_TOL = 2e-13   # measured 1.3e-14
SOLVE_TOL = 3e-15    # measured 5.8e-17 (the blocks are 1 x 1 and 2 x 2)
DOT_TOL = 5e-14      # measured 1.7e-15
DENSE_BLOCK_RTOL = 4e-15   # a dense-fallback block against the oracle's kernel values; zeros must be exact

BIG = dict(n=262147, min_size=512)      # root of 131074 rows: about two Lemire rejections per scan
MEDIUM = dict(n=65539, min_size=256)    # nodes of 32770, 16385, 8192, 4096 rows: batches of 8192 that collide with themselves
SMALL = dict(n=4001, min_size=60)       # dense fallback blocks stay small


@pytest.fixture
def clean_env(monkeypatch):
    for var in ("BGP_NO_GRAPH", "BGP_NO_CULL", "BGP_EVAL_MINB"):
        monkeypatch.delenv(var, raising=False)
    return monkeypatch


def _rows(P, node):
    nd = P.nodes[node]
    return nd["size"] - nd["half"]


def _group(P, node, size, pos, terminate, sub_threshold=True):
    """Reject whole batches until one of `size` candidates is pending, then a winner at `pos` of it (negative: from the
    end), two more accepts right behind it, and either a terminator or nothing (the node then runs out of rows)."""
    d = P.draws(node)
    s = M.Schedule(_rows(P, node), d.rejected).reject_until(size=size)
    c = s.accept(pos % size)
    if sub_threshold and c >= 1:
        P.place(node, c - 1, M.SUB_THRESHOLD, d)
    P.place(node, c, M.NORMAL[node % 4], d)
    P.place(node, c + 1, M.NORMAL[(node + 1) % 4], d)
    P.place(node, c + 2, M.NORMAL[(node + 2) % 4], d)
    if terminate:
        P.place(node, c + 6, M.TERMINATOR if node % 2 else M.AT_THRESHOLD, d)
        P.place(node, c + 20, 0.9, d)   # never visited: dropped from K_h
    return c


def _medium(seed_index, **kw):
    seed = (42, 7, 1234)[seed_index]
    P = M.Problem(seed=seed, **dict(MEDIUM, **kw))
    big = [i for i, nd in enumerate(P.nodes) if not nd["is_leaf"] and _rows(P, i) >= 10532]
    mid = [i for i, nd in enumerate(P.nodes) if not nd["is_leaf"] and 4096 <= _rows(P, i) < 10532]
    assert len(big) == 3 and len(mid) == 12
    positions = (0, 1, -2, -1)
    for k, node in enumerate(big):
        _group(P, node, 8192, positions[(k + seed_index) % 4], terminate=(k + seed_index) % 2 == 0)
    combos = [(size, pos) for size in (32, 256, 2048) for pos in positions]
    for k, node in enumerate(mid):
        size, pos = combos[(k + 5 * seed_index) % 12]
        _group(P, node, size, pos, terminate=k % 2 == 0)
    return P


def _small(seed=42, **kw):
    P = M.Problem(seed=seed, **dict(SMALL, **kw))
    inner = [i for i, nd in enumerate(P.nodes) if not nd["is_leaf"] and _rows(P, i) >= 400]
    sizes = {2001: (1709, 800), 2000: (256, -2), 1001: (256, 0), 1000: (32, 1), 501: (32, -1), 500: (32, 0)}
    for k, node in enumerate(inner):
        size, pos = sizes.get(_rows(P, node), (32, 1))
        _group(P, node, size, pos, terminate=k % 2 == 1)
    return P


# ---- Lemire rejections in the root of the BIG problem: (seed, recipe) found by tools/find_draw_seeds.py ------------
def _big(seed, recipe):
    P = M.Problem(seed=seed, **BIG)
    d = P.draws(0)
    n_rows = _rows(P, 0)
    s = M.Schedule(n_rows, d.rejected)
    rej = [r for r in d.rejected if r >= 2340]
    r = rej[0] if rej else None
    expect = {"lemire_redos": 1}
    if recipe == "before":       # the winner comes after the rejection in its batch: its row depends on the shifted offset
        s.reject_until(draw=r)
        assert s.first + s.size() > r + 6
        P.place(0, r + 1, M.SUB_THRESHOLD, d)
        P.place(0, s.accept(r + 2 - s.first), 0.5, d)
        P.place(0, r + 5, M.TERMINATOR, d)
        expect["partial_commits"] = 1
    elif recipe == "after":      # the node stops before a rejection of the same batch: it is not counted
        P.place(0, s.accept(2), 0.5, d)
        s.reject_until(draw=r - 2)
        assert s.first + s.size() > r
        P.place(0, r - 2, M.AT_THRESHOLD, d)
        expect["partial_commits"] = 1
    elif recipe == "two":        # two rejections in one batch, the winner behind both
        r, r2 = next((a, b) for a, b in zip(rej, rej[1:]) if a != b and (a - 2340) // 8192 == (b - 2340) // 8192)
        s.reject_until(draw=r)
        assert s.first + s.size() > r2 + 6
        P.place(0, s.accept(r2 + 2 - s.first), 0.6, d)
        P.place(0, r2 + 5, M.TERMINATOR, d)
        expect = {"lemire_redos": 2, "partial_commits": 1}
    elif recipe == "draw0":      # an accept just before the rejection: it is draw 0 of the next batch
        P.place(0, s.accept_draw(r - 1), 0.7, d)
        assert s.first == r
        P.place(0, r + 1, M.TERMINATOR, d)
    elif recipe == "last":       # an accept that makes the rejection the last draw of the next batch: the batch is truncated
        def start(q):
            return M.Schedule(n_rows, d.rejected).reject_until(draw=q).first
        r = next(q for q in rej if (q - start(q) - 2) % 3 == 0 and q - start(q) >= 5)
        s.reject_until(draw=r)
        P.place(0, s.accept((r - s.first - 2) // 3), 0.8, d)
        assert s.first + s.size() == r and r in s.rejected
        s.reject()
        assert s.first == r
        P.place(0, r + 2, 0.5, d)
        P.place(0, r + 4, M.TERMINATOR, d)
        expect["truncated_batches"] = 1
    elif recipe == "full":       # a rejection in a fully consumed batch, the winner in a later one; then the rows run out
        s.reject_until(draw=r)
        s.reject()
        P.place(0, s.accept(100), 0.5, d)
        P.place(0, s.first + 3, 0.6, d)
    elif recipe == "single":     # the first rows are all usable, so batches hold ONE candidate, and one of them rejects a word
        r = d.rejected[0]
        assert r < 60
        for c in range(r + 2):
            P.place(0, c, M.NORMAL[c % 4], d)
        expect["sequential_draws"] = 1
    else:
        raise ValueError(recipe)
    return P, expect


def _compute(P, solver=None, exhaust="lowrank", rng_mode="pernode"):
    from george_b200.solvers._hodlr import HODLRSolver
    s = solver or HODLRSolver()
    s.compute(P.kernel(), P.x, YERR * np.ones(P.n), min_size=P.min_size, tol=P.tol, seed=P.seed, rng_mode=rng_mode,
              exhaust=exhaust, rank_capacity=0 if exhaust == "dense" else 64)   # (dense blocks need their full rank)
    return s


def _check_decisions(P, s, pred, exhaust):
    """Every internal node: rank, pivot rows and columns, words drawn and the exhaustion flag equal the model."""
    nodes = s.nodes()
    assert [(nd["start"], nd["size"], nd["half"], bool(nd["is_leaf"])) for nd in nodes] == \
        [(nd["start"], nd["size"], nd["half"], nd["is_leaf"]) for nd in P.nodes]
    for i, nd in enumerate(nodes):
        if nd["is_leaf"]:
            continue
        p = pred[i]
        dense = exhaust == "dense" and p["dense_fallback"]
        rank = min(nd["half"], nd["size"] - nd["half"]) if dense else p["rank"]
        got = (nd["rank"], nd["rng_draws"], nd["dense_fallback"])
        assert got == (rank, p["rng_draws"], p["dense_fallback"]), (i, nd, got, p["rows"], p["draws"].rejected)
        if not dense:
            rows, cols = s.pivots(i, nd["rank"])
            assert list(rows) == p["rows"] and list(cols) == p["cols"], (i, list(rows), p["rows"], list(cols), p["cols"])


def _check_numerics(P, s, pred, exhaust, record_property):
    d = np.float64(1.0) + np.float64(YERR) ** 2
    ref = M.BlockReference(P.n, d, P.kept_pairs(pred, exhaust))
    rng = np.random.default_rng(P.seed + P.n)
    B = rng.normal(size=(P.n, 65))
    errs = {"logdet": abs(s.log_determinant - ref.logdet) / max(1.0, abs(ref.logdet))}
    for cols in (B[:, 0], B):
        X, Xr = np.asarray(s.apply_inverse(cols), dtype=LD).reshape(cols.shape), ref.solve(cols)
        errs["solve%d" % (cols.shape[1] if cols.ndim == 2 else 1)] = float(np.sqrt(np.sum((X - Xr) ** 2) / np.sum(Xr ** 2)))
    y = B[:, 1]
    q_ref = float(np.dot(y.astype(LD), ref.solve(y)))
    errs["dot_solve"] = abs(s.dot_solve(y) - q_ref) / abs(q_ref)
    for k, v in errs.items():
        record_property(k, v)
    assert errs["logdet"] <= LOGDET_TOL and errs["dot_solve"] <= DOT_TOL, errs
    assert max(errs["solve1"], errs["solve65"]) <= SOLVE_TOL, errs


def _check_dense_blocks(P, s, pred, oracle):
    """exhaust = "dense": a node that ran out of rows stores its block itself (V = I, U = K[right, left])."""
    from george_b200._spec import flatten
    spec, x = flatten(P.kernel()), P.x
    for i, nd in enumerate(P.nodes):
        if nd["is_leaf"] or not pred[i]["dense_fallback"]:
            continue
        lo, mid, hi = nd["start"], nd["start"] + nd["half"], nd["start"] + nd["size"]
        Vl, Ur = s.factors(i)
        Kb = oracle.value_general(spec, x[mid:hi], x[lo:mid])
        assert np.count_nonzero(Kb) == len(P.pairs.get(i, []))
        assert np.array_equal(Vl, np.eye(nd["half"]))
        assert np.array_equal(Ur == 0.0, Kb == 0.0), i
        np.testing.assert_allclose(Ur, Kb, rtol=DENSE_BLOCK_RTOL, atol=0.0)


def _run(P, record_property, expect=None, exhaust="lowrank", solver=None, rng_mode="pernode", oracle=None):
    pred = P.predict()
    s = _compute(P, solver=solver, exhaust=exhaust, rng_mode=rng_mode)
    paths = s.draw_paths()
    record_property("draw_paths", paths)
    _check_decisions(P, s, pred, exhaust)
    for name, least in (expect or {}).items():
        assert paths[name] >= least, (name, paths)
    if exhaust == "dense":
        _check_dense_blocks(P, s, pred, oracle)
    _check_numerics(P, s, pred, exhaust, record_property)
    return s, pred, paths


@pytest.mark.parametrize("seed_index", [0, 1, 2])
def test_accepts_inside_large_batches(gpu, clean_env, record_property, seed_index):
    """A winner at positions 0, 1, B-2 and B-1 of batches of 32, 256, 2048 and 8192 after a long rejected run, with a
    rejected sub-threshold row just before it and two more accepts behind it; half of the nodes then stop on a
    terminator in the middle of a batch, the others run out of rows.  The batches of 8192 on the lists of 16385 rows
    collide with themselves heavily, so the rows come through the writer chains of the swap-pop."""
    _run(_medium(seed_index), record_property, expect={"partial_commits": 15})


BIG_CASES = [(3, "before"), (8, "before"), (3, "after"), (9, "after"), (2, "two"), (74, "two"), (3, "draw0"),
             (8, "draw0"), (3, "last"), (8, "last"), (9, "last"), (3, "full"), (9, "full"), (640, "single"),
             (2658, "single")]


@pytest.mark.parametrize("seed,recipe", BIG_CASES)
def test_lemire_rejection_paths(gpu, clean_env, record_property, seed, recipe):
    """A Lemire rejection in the root's scan of 131074 rows: before the winner of its batch, after it, twice in one
    batch, at draw 0 of a batch, at the last draw (the batch is truncated), in a fully consumed batch, and in a
    one-candidate batch (drawn sequentially)."""
    P, expect = _big(seed, recipe)
    _run(P, record_property, expect=expect)


@pytest.mark.parametrize("exhaust", ["lowrank", "dense"])
def test_exhaustion_small(gpu, clean_env, oracle, record_property, exhaust):
    """Both exhaustion modes where the dense blocks are small: a node that runs out of rows after its last special row
    drew n_rows words (no rejection at these sizes) and, in dense mode, stores its block entry for entry."""
    P = _small()
    _, pred, _ = _run(P, record_property, exhaust=exhaust, oracle=oracle)
    out = [i for i in P.pairs if pred[i]["dense_fallback"]]
    assert len(out) >= 3 and all(pred[i]["rng_draws"] == _rows(P, i) and pred[i]["rank"] == 3 for i in out)


@pytest.mark.parametrize("route", ["no_cull", "ndim2", "no_graph"])
def test_every_evaluation_route_takes_the_same_decisions(gpu, clean_env, record_property, route):
    """1-D with bound culling is the default above (the moved partners stretch a node's column box, so culled and live
    candidates mix); here the exhaustive 1-D scan, 2-D inputs through the general interpreter, and the host-driven
    loop."""
    if route == "no_cull":
        clean_env.setenv("BGP_NO_CULL", "1")
    if route == "no_graph":
        clean_env.setenv("BGP_NO_GRAPH", "1")
    _run(_medium(0, ndim=2 if route == "ndim2" else 1), record_property, expect={"partial_commits": 15})


@pytest.mark.parametrize("seed", [862, 4283])   # (with 16 two nodes of this construction want the same row)
def test_chained_reference_stream(gpu, clean_env, record_property, seed):
    """rng_mode = "reference" (aca_kernel, one stream through the tree in pre-order) with a Lemire rejection in the
    root's scan before its winner: every later node starts at an offset that counts the rejected word."""
    P = M.Problem(n=8193, min_size=128, seed=seed, chained=True)
    d = P.draws(0)
    r = d.rejected[0]
    P.place(0, r + 3, 0.5, d)
    P.place(0, r + 9, M.TERMINATOR, d)
    for node in [i for i, nd in enumerate(P.nodes) if not nd["is_leaf"] and _rows(P, i) >= 1024][1:]:
        _group(P, node, 256, (0, 1, -2, -1)[node % 4], terminate=node % 2 == 0)
    pred = P.predict()
    assert pred[0]["rng_draws"] == r + 9 + 2
    _, _, paths = _run(P, record_property, rng_mode="reference")
    assert not any(paths.values())   # one row at a time: no speculation


def test_handle_reuse(gpu, clean_env, oracle, record_property):
    """One native handle runs steered problems of different sizes and seeds in turn: candidate buffers, the row lists
    and the cached ACA graph of the previous problem must not leak into the next."""
    from george_b200.solvers._hodlr import HODLRSolver
    HODLRSolver.release_parked()
    s = HODLRSolver()
    for P, exhaust in ((_medium(1), "lowrank"), (_small(7), "dense"), (_medium(2), "lowrank"), (_small(42), "lowrank"),
                       (_medium(1), "lowrank")):
        _run(P, record_property, exhaust=exhaust, solver=s, oracle=oracle)
    del s
    HODLRSolver.release_parked()
