# -*- coding: utf-8 -*-
"""The sharded variance gradient on CPU: ShardedHODLRSolver.predictive_grad's presence, its check before compute, the
buffers it hands to bgp_hodlr_predict_grad (with the native handle replaced by a stand-in that records the call), and
the ctypes signature of bgp_hodlr_predict_grad_local_dev against include/bgp.h.  The collective arithmetic needs several
GPUs (tools/mgpu_check.py); one shard's part runs on one GPU in tests/test_gpu_hodlr_shard_predict_grad.py."""
import ctypes as C
import os
import re

import numpy as np
import pytest

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "bgp.h")


class _FakeLib(object):
    """bgp_hodlr_predict_grad: records (ptr, ndim, xs, ns) and writes var[j] = j, dvar[k] = 1000 + k."""

    def __init__(self):
        self.calls = []

    def bgp_hodlr_predict_grad(self, ptr, spec, xs, ns, var, dvar):
        ndim = spec._obj.ndim
        xv = [C.cast(xs, C.POINTER(C.c_double))[i] for i in range(ns * ndim)]
        self.calls.append((ptr, ndim, xv, ns))
        v, d = C.cast(var, C.POINTER(C.c_double)), C.cast(dvar, C.POINTER(C.c_double))
        for j in range(ns):
            v[j] = float(j)
        for k in range(ns * ndim):
            d[k] = 1000.0 + k
        return 0


class _FakeNative(object):
    def __init__(self):
        self._lib = _FakeLib()
        self._ptr = C.c_void_p(4321)


def _solver(computed=True):
    from george_b200 import kernels
    from george_b200.parallel import ShardedHODLRSolver
    s = ShardedHODLRSolver(1.0 * kernels.ExpKernel(1.0))
    if computed:
        s.solver = _FakeNative()
        s._n = 10
        s._computed = True
    return s


def _kernel(ndim=1):
    from george_b200 import kernels
    return 1.5 * kernels.Matern32Kernel(0.7, ndim=ndim)


def test_predictive_grad_exists():
    from george_b200.parallel import ShardedHODLRSolver
    assert callable(getattr(ShardedHODLRSolver, "predictive_grad", None))


def test_predictive_grad_before_compute_raises():
    with pytest.raises(RuntimeError, match="compute"):
        _solver(computed=False).predictive_grad(_kernel(), np.zeros((3, 1)))


def test_predictive_grad_rejects_a_kernel_of_another_dimension():
    from george_b200._spec import DimensionMismatch
    s = _solver()
    with pytest.raises(DimensionMismatch):
        s.predictive_grad(_kernel(2), np.zeros((3, 1)))
    assert s.solver._lib.calls == []


def test_predictive_grad_shapes_and_buffers():
    """var (ns,) and dvar (ns, ndim), float64; xs converted to contiguous float64 rows."""
    s = _solver()
    xs = np.asfortranarray(np.arange(6, dtype=np.int32).reshape(3, 2))
    var, dvar = s.predictive_grad(_kernel(2), xs)
    assert var.dtype == dvar.dtype == np.float64 and var.shape == (3,) and dvar.shape == (3, 2)
    assert np.array_equal(var, np.arange(3.0)) and np.array_equal(dvar.ravel(), 1000.0 + np.arange(6))
    (ptr, ndim, xv, ns), = s.solver._lib.calls
    assert ptr.value == 4321 and ndim == 2 and ns == 3 and xv == [0.0, 1.0, 2.0, 3.0, 4.0, 5.0]
    var, dvar = s.predictive_grad(_kernel(), np.zeros(0))
    assert var.shape == (0,) and dvar.shape == (0, 1)


def _declared_params(name):
    """The parameter types of `name`'s declaration in include/bgp.h, without the parameter names."""
    with open(HEADER) as f:
        text = f.read()
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", text)
    assert m is not None, name
    params = [" ".join(p.split()) for p in m.group(1).split(",")]
    return [re.sub(r"\s*\b\w+$", "", p) for p in params]


def test_local_entry_signature_matches_the_header():
    from george_b200 import _lib
    from george_b200._spec import KernelSpec
    ctype = {"bgp_hodlr_t*": C.c_void_p, "const bgp_kernel_spec_t*": C.POINTER(KernelSpec),
             "const double*": C.c_void_p, "double*": C.c_void_p, "int64_t": C.c_int64, "int32_t": C.c_int32}
    name = "bgp_hodlr_predict_grad_local_dev"
    declared = _declared_params(name)
    assert declared == ["bgp_hodlr_t*", "const bgp_kernel_spec_t*", "const double*", "int64_t", "const double*",
                        "int64_t", "int32_t", "double*", "double*"]
    res, args = _lib.SIGNATURES[name]
    assert res is C.c_int
    assert args == [ctype[t] for t in declared]
