# -*- coding: utf-8 -*-
"""The oracle's ACA on NaN rows (oracle/hodlr_oracle.cpp: low_rank_approx), held to pivots worked out by hand.

The rule every ACA route follows (DESIGN.md §2): in a row's arg-max a NaN counts as +inf, so the first NaN in column
order wins, and a NaN pivot is accepted.  The blocks are ExpSquaredKernel(1.0) on points 64 length scales apart, so
every off-diagonal entry is exactly 0 except the pairs moved next to each other; the draw order of the root's rows comes
from the independent model in tests/aca_draw_model.py.
"""
import numpy as np
import pytest

import aca_draw_model as M

N, MIN_SIZE, SEED = 8, 4, 42   # root: block rows 4..7 against columns 0..3; the children are leaves


def _root_draws():
    return M.Draws(M.mt19937_words(M.node_seed(SEED, 0), M.words_needed(N // 2)), N // 2).rows.tolist()


def _root(oracle, x):
    from george_b200 import kernels
    from george_b200._spec import flatten
    h = oracle.HODLR(flatten(kernels.ExpSquaredKernel(1.0)), x, 0.1 * np.ones(N), min_size=MIN_SIZE, tol=1e-10,
                     seed=SEED, rng_mode=1, exhaust=1)
    root = h.nodes()[0]
    rows, cols = h.pivots(0, root["rank"])
    return root, list(rows), list(cols)


@pytest.mark.parametrize("nan_col", [1, 2, 3])
def test_partly_nan_row_pivots_on_its_first_nan(oracle, nan_col):
    """The first row drawn is 0.5 at column 0, a NaN at `nan_col` and 0 elsewhere: the NaN wins over the larger finite
    entry.  Its normalised row is all NaN, so every later row is all NaN and pivots on column 0 until the node reaches
    full rank."""
    draws = _root_draws()
    x = M.SPACING * np.arange(N, dtype=np.float64)
    r = draws[0]
    x[0] = x[N // 2 + r] + np.sqrt(-2.0 * np.log(0.5))   # K(row r, column 0) = 0.5
    x[nan_col] = np.nan
    root, rows, cols = _root(oracle, x)
    assert (root["rank"], root["dense_fallback"]) == (4, 0)
    assert rows == draws and cols == [nan_col, 0, 0, 0]


def test_all_nan_row_pivots_on_column_zero(oracle):
    """The first row drawn has one sub-threshold entry at column 3 (rejected: its arg-max is 3); the second is all NaN
    (its point is NaN) and pivots on column 0, not on the column the rejected row left behind."""
    draws = _root_draws()
    x = M.SPACING * np.arange(N, dtype=np.float64)
    x[3] = x[N // 2 + draws[0]] + 8.2   # K = exp(-0.5 * 8.2^2) = 2.4e-15 < 1e-14
    x[N // 2 + draws[1]] = np.nan
    root, rows, cols = _root(oracle, x)
    # three rows accepted, then the list is empty: exhaust = 1 keeps the low-rank factors
    assert (root["rank"], root["dense_fallback"], root["rng_draws"]) == (3, 1, 4)
    assert rows == draws[1:] and cols == [0, 0, 0]


def test_finite_rows_keep_the_largest_entry(oracle):
    """Without a NaN the rule is the old one: the largest |entry| wins."""
    draws = _root_draws()
    x = M.SPACING * np.arange(N, dtype=np.float64)
    r = draws[0]
    x[1] = x[N // 2 + r] - np.sqrt(-2.0 * np.log(0.5))
    x[2] = x[N // 2 + r] + np.sqrt(-2.0 * np.log(0.7))
    root, rows, cols = _root(oracle, x)
    assert rows[0] == r and cols[0] == 2
