# -*- coding: utf-8 -*-
"""
Generates tests/golden/reference_kernel_interface.json: SHA-256 digests (golden_digest below) of what the reference's OWN
compiled kernel_interface.cpp (oracle/_ref, built by `make -C oracle ref` from the reference sources) returns for every
kernel of the zoo in tests/conftest.py (make_kernels), of the reference's own kernel suite (reference_kernel_list) and
of the size-limit programs of tests/test_gpu_program_limits.py (limit_programs), on the inputs that
tests/test_oracle_kernels.py, tests/test_reference_kernel_list.py and tests/test_gpu_program_limits.py draw.  Those tests compare the
CPU oracle with the reference bit for bit through these digests, so they run wherever the repository is checked out.
(Digests rather than the arrays: the outputs are ~0.9 MB of incompressible doubles.)

Run from the repo root:   python tests/golden/make_golden_kernel_interface.py     (needs `make -C oracle ref`)
"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
PATH = os.path.join(HERE, "reference_kernel_interface.json")


def golden_digest(a):
    """Digest of the shape and the exact float64 bits (-0.0 counted as +0.0, which np.array_equal also equates)."""
    a = np.ascontiguousarray(a, dtype=np.float64) + 0.0
    assert not np.isnan(a).any()
    return hashlib.sha256(repr(a.shape).encode() + a.tobytes()).hexdigest()


def main():
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.dirname(HERE))
    import oracle
    from conftest import make_kernels, reference_kernel_list
    ref = oracle.reference_kernel_interface()
    assert ref is not None, "run `make -C oracle ref` first"
    out = {}
    for name, kernel in make_kernels():  # tests/test_oracle_kernels.py::test_oracle_equals_reference_binary
        rng = np.random.default_rng(1)
        nd = kernel.ndim
        x1, x2 = rng.normal(size=(31, nd)), rng.normal(size=(19, nd))
        r = ref.KernelInterface(kernel)
        p = "zoo__" + name + "__"
        out[p + "value_general"] = r.value_general(x1, x2)
        out[p + "value_symmetric"] = r.value_symmetric(x1)
        out[p + "value_diagonal"] = r.value_diagonal(x1[:19], x2)
        if kernel.full_size:
            out[p + "gradient_general"] = r.gradient_general(np.ones(kernel.full_size, dtype=np.uint32), x1, x2)
    for i, kernel in enumerate(reference_kernel_list()):  # tests/test_reference_kernel_list.py
        np.random.seed(123)
        t1 = np.random.randn(20, kernel.ndim)
        r = ref.KernelInterface(kernel)
        p = "list__{0:02d}__".format(i)
        out[p + "value_symmetric"] = r.value_symmetric(t1)
        out[p + "value_general"] = r.value_general(t1, t1[:1])
        if kernel.full_size:
            out[p + "gradient_general"] = r.gradient_general(np.ones(kernel.full_size, dtype=np.uint32), t1, t1[:3])
        out[p + "x1_gradient_general"] = r.x1_gradient_general(t1, t1[:3])
        out[p + "x2_gradient_general"] = r.x2_gradient_general(t1[:3], t1)
    from test_gpu_program_limits import reference_outputs  # tests/test_gpu_program_limits.py: the size limits
    out.update(reference_outputs(ref))
    with open(PATH, "w") as fh:
        json.dump({k: golden_digest(v) for k, v in out.items()}, fh, indent=0, sort_keys=True)
        fh.write("\n")
    print("wrote", PATH, "with", len(out), "digests")


if __name__ == "__main__":
    main()
