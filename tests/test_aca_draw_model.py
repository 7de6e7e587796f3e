# -*- coding: utf-8 -*-
"""tests/aca_draw_model.py against the real libstdc++ (std::mt19937, std::uniform_int_distribution<int>) through the
oracle, on the seeds tests/test_gpu_hodlr_draws.py hard-codes; and those seeds have the properties its cases rely on.
No GPU needed."""

import numpy as np
import pytest

import aca_draw_model as M

BIG_ROWS = 262147 - 262147 // 2
# seed -> the rejecting draws of the root's scan of BIG_ROWS rows (tools/find_draw_seeds.py)
BIG_SEEDS = [2, 3, 8, 9, 74, 640, 2658]
CHAINED_SEEDS = {16: 301, 862: 1146, 4283: 770}   # first rejecting draw of a scan of 4097 rows


@pytest.mark.parametrize("seed", [0, 42, 5489, 4294967295])
def test_words_are_mt19937(oracle, seed):
    assert np.array_equal(M.mt19937_words(seed, 1500), oracle.mt19937_words(seed, 1500))
    assert M.node_seed(seed, 3) == (seed + 3 * 0x9E3779B9) % 2 ** 32


@pytest.mark.parametrize("seed,n_rows", [(s, BIG_ROWS) for s in BIG_SEEDS] + [(s, 4097) for s in CHAINED_SEEDS]
                         + [(5, 2 ** 18 + 1), (6, 2 ** 18), (42, 10000)])
def test_draws_are_libstdcxx(oracle, seed, n_rows):
    """Every draw of a whole scan, rejections included: the same positions as libstdc++ draws from the same seed."""
    d = M.Draws(M.mt19937_words(seed, M.words_needed(n_rows)), n_rows)
    assert np.array_equal(d.k, oracle.uniform_ints(seed, np.arange(n_rows, 0, -1)))
    assert d.cum[-1] == n_rows + len(d.rejected)
    assert np.array_equal(np.sort(d.rows), np.arange(n_rows))   # the swap-pop visits every row once
    if n_rows != 10000:
        assert d.rejected, "this size and seed were chosen because the scan rejects a word"
        # the words the model says were consumed are the ones libstdc++ consumed: drawing one more value afterwards
        # from a stream of exactly cum[-1] skipped words gives the same number on both sides
        sizes = np.concatenate([np.arange(n_rows, 0, -1), [1000003]])
        tail = oracle.uniform_ints(seed, sizes)[-1]
        w = M.mt19937_words(seed, int(d.cum[-1]) + 8)[int(d.cum[-1]):]
        assert M.uniform_draws(w, [1000003])[0][0] == tail


def test_seed_properties():
    """What the steered GPU cases need from their hard-coded seeds."""
    def rejected(seed, n_rows=BIG_ROWS):
        return M.Draws(M.mt19937_words(seed, M.words_needed(n_rows)), n_rows, order=False).rejected

    def start(draw):   # of the fully rejected batch of 8192 holding `draw`
        return 2340 + (draw - 2340) // 8192 * 8192
    for seed in (3, 8, 9):     # a rejection that one accept turns into the last draw of a batch
        assert any(r >= 2340 and r - start(r) >= 5 and (r - start(r) - 2) % 3 == 0 for r in rejected(seed)), seed
    for seed in (2, 74):       # two rejections in one batch of 8192
        rej = rejected(seed)
        assert any(a != b and a >= 2340 and start(a) == start(b) for a, b in zip(rej, rej[1:])), seed
    for seed in (640, 2658):   # a rejection within the first rows, reachable with one-candidate batches
        assert 4 <= rejected(seed)[0] < 60, seed
    for seed, first in CHAINED_SEEDS.items():
        assert rejected(seed, 4097)[0] == first


@pytest.mark.parametrize("chained", [False, True])
def test_prediction_equals_oracle_on_a_constructed_problem(oracle, chained):
    """The whole prediction (ranks, pivot rows and columns, draws, exhaustion) against the oracle's low_rank_approx on a
    partial-permutation problem whose root rejects a word before its winner.  The oracle counts draws, the model (like
    the device) words: they differ by the rejections up to the last draw consumed."""
    from george_b200._spec import flatten
    seed = 16
    P = M.Problem(n=8193, min_size=512, seed=seed, chained=chained)
    d = P.draws(0)
    r = d.rejected[0]
    P.place(0, r + 1, M.SUB_THRESHOLD, d)
    P.place(0, r + 3, 0.5, d)
    P.place(0, r + 9, M.TERMINATOR, d)
    P.place(0, r + 30, 0.9, d)
    for node in [i for i, nd in enumerate(P.nodes) if not nd["is_leaf"]][1:4]:
        dn = P.draws(node)
        P.place(node, 40, 0.6, dn)
        P.place(node, 41, M.AT_THRESHOLD if node % 2 else 0.7, dn)
    pred = P.predict()
    assert pred[0]["rank"] == 2 and pred[0]["rng_draws"] == r + 11 and not pred[0]["dense_fallback"]
    o = oracle.HODLR(flatten(P.kernel()), P.x, 0.1 * np.ones(P.n), min_size=P.min_size, tol=P.tol, seed=seed,
                     rng_mode=1 if chained else 0, exhaust=1)
    on = o.nodes()
    assert [(nd["start"], nd["size"], nd["half"], bool(nd["is_leaf"])) for nd in on] == \
        [(nd["start"], nd["size"], nd["half"], nd["is_leaf"]) for nd in P.nodes]
    for i, nd in enumerate(on):
        if nd["is_leaf"]:
            continue
        p = pred[i]
        words = nd["rng_draws"] + p["draws"].rejections_up_to(nd["rng_draws"] - 1)
        assert (nd["rank"], words, nd["dense_fallback"]) == (p["rank"], p["rng_draws"], p["dense_fallback"]), (i, nd, p)
        rows, cols = o.pivots(i, nd["rank"])
        assert list(rows) == p["rows"] and list(cols) == p["cols"], i
    # K_h in closed form against the oracle's factorisation
    ref = M.BlockReference(P.n, np.float64(1.0) + np.float64(0.1) ** 2, P.kept_pairs(pred, "lowrank"))
    assert abs(o.log_determinant - ref.logdet) <= 1e-12 * abs(ref.logdet)
    y = np.sin(np.arange(P.n))
    assert np.allclose(o.apply_inverse(y), np.asarray(ref.solve(y), dtype=np.float64), rtol=1e-12, atol=0)
