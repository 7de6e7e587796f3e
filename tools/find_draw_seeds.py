# -*- coding: utf-8 -*-
"""Deterministic search for the seeds hard-coded in tests/test_gpu_hodlr_draws.py: root nodes whose Lemire rejections
fall where a steered case needs them.  tests/test_aca_draw_model.py re-verifies every property printed here.

    python tools/find_draw_seeds.py
"""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
import aca_draw_model as M  # noqa: E402
import numpy as np  # noqa: E402


def rejections(seed, n_rows, first=None):
    m = n_rows if first is None else first
    w = M.mt19937_words(seed, m + 64)
    return M.uniform_draws(w, np.arange(n_rows, n_rows - m, -1))[2]


def full_batch_start(draw):
    """Start of the fully rejected batch of 8192 that holds `draw` when nothing was accepted before it."""
    return 2340 + (draw - 2340) // 8192 * 8192 if draw >= 2340 else None


def last_draw_recipe(rej):
    """A rejection r that an accept at position p of its batch turns into the LAST draw of the next batch:
    start + p + 1 + 2 (p + 1) - 1 = r."""
    for r in rej:
        f0 = full_batch_start(r)
        if f0 is not None and r - f0 >= 5 and (r - f0 - 2) % 3 == 0:
            return r
    return None


def two_in_one_batch(rej):
    for r1, r2 in zip(rej, rej[1:]):
        if r1 != r2 and full_batch_start(r1) is not None and full_batch_start(r1) == full_batch_start(r2):
            return r1, r2
    return None


if __name__ == "__main__":
    big = 262147 - 262147 // 2
    found = {"last": [], "two": [], "early": [], "chained": []}
    for seed in range(200):
        rej = rejections(seed, big)
        if len(found["last"]) < 3 and last_draw_recipe(rej) is not None:
            found["last"].append((seed, last_draw_recipe(rej)))
        if len(found["two"]) < 2 and two_in_one_batch(rej):
            found["two"].append((seed, two_in_one_batch(rej)))
    for seed in range(200000):
        if len(found["early"]) < 2:
            rej = rejections(seed, big, first=40)
            if rej and 4 <= rej[0]:
                found["early"].append((seed, rej[0]))
        if len(found["chained"]) < 8:
            rej = rejections(seed, 8193 - 8193 // 2)
            if rej:
                found["chained"].append((seed, rej[0]))
        if len(found["early"]) == 2 and len(found["chained"]) == 8:
            break
    for k, v in found.items():
        print(k, v)
