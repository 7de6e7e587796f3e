# -*- coding: utf-8 -*-
"""
Bits of the panel-by-panel leaf LDL^T kernel, for tests/test_gpu_hodlr_leaf_lookahead.py.

    python tests/golden/make_golden_leaf_factor.py        (on an H100, with the library built from a tree whose
                                                           leaf_factor_kernel has no lookahead: 4817194 and before)

For every case of the test (a single-leaf tree: the leaf is the whole LDL^T of K) it stores the log-determinant, two
solves and the symmetric factor applied to a vector, float64.  The lookahead kernel keeps each entry's summation order,
so it must reproduce them bit for bit.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))  # the package
sys.path.insert(0, os.path.dirname(HERE))  # the test module and its helpers
import test_gpu_hodlr_leaf_lookahead as t  # noqa: E402

os.environ.pop("BGP_LEAF_FACTOR", None)
os.environ.pop("BGP_LEAF_COLS", None)
out = {}
for kname, n in t.CASES:
    s = t.single_leaf(kname, n)[0]
    for key, v in t.leaf_outputs(s, n).items():
        out["{0}_{1}_{2}".format(kname, n, key)] = v
path = os.path.join(HERE, "leaf_factor_bits.npz")
np.savez_compressed(path, **out)
print(len(out), "arrays ->", path)
