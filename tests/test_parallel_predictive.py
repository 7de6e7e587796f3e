# -*- coding: utf-8 -*-
"""ShardedHODLRSolver.predictive on CPU: its argument checks, output shapes and the buffers it hands to
bgp_hodlr_predict, with the native handle replaced by a stand-in that records the call and fills the output.  The
collective arithmetic itself needs several GPUs (tools/mgpu_check.py); one shard's part runs on one GPU in
tests/test_gpu_hodlr_shard_predict.py."""
import ctypes as C

import numpy as np
import pytest


class _FakeLib(object):
    """bgp_hodlr_predict: records (ptr, ndim, xs, ns, what) and writes out[k] = 100 * what + k."""

    def __init__(self):
        self.calls = []

    def bgp_hodlr_predict(self, ptr, spec, xs, ns, what, out):
        ndim = spec._obj.ndim
        xv = [C.cast(xs, C.POINTER(C.c_double))[i] for i in range(ns * ndim)]
        self.calls.append((ptr, ndim, xv, ns, what))
        o = C.cast(out, C.POINTER(C.c_double))
        for k in range(ns if what == 0 else ns * ns):
            o[k] = 100.0 * what + k
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


def test_predictive_before_compute_raises():
    with pytest.raises(RuntimeError, match="compute"):
        _solver(computed=False).predictive(_kernel(), np.zeros((3, 1)), "var")


def test_predictive_rejects_an_unknown_kind():
    s = _solver()
    with pytest.raises(ValueError, match="'var' or 'cov'"):
        s.predictive(_kernel(), np.zeros((3, 1)), "mean")
    assert s.solver._lib.calls == []


def test_predictive_rejects_a_kernel_of_another_dimension():
    from george_b200._spec import DimensionMismatch
    s = _solver()
    with pytest.raises(DimensionMismatch):
        s.predictive(_kernel(2), np.zeros((3, 1)), "cov")
    assert s.solver._lib.calls == []


@pytest.mark.parametrize("what,kind", [("var", 0), ("cov", 1)])
def test_predictive_shapes_and_buffers(what, kind):
    """(ns,) or (ns, ns) float64; 1-D xs become a column, converted to contiguous float64 rows."""
    s = _solver()
    xs = np.arange(4, dtype=np.int32)  # converted to float64, one column
    out = s.predictive(_kernel(), xs, what)
    ns = 4
    assert out.dtype == np.float64 and out.shape == ((ns,) if what == "var" else (ns, ns))
    assert np.array_equal(out.ravel(), 100.0 * kind + np.arange(out.size))
    (ptr, ndim, xv, n_s, w), = s.solver._lib.calls
    assert ptr.value == 4321 and ndim == 1 and n_s == ns and w == kind and xv == [0.0, 1.0, 2.0, 3.0]


def test_predictive_row_major_points_in_several_dimensions():
    s = _solver()
    xs = np.asfortranarray(np.arange(6, dtype=np.float64).reshape(3, 2))  # made C-contiguous on the way
    out = s.predictive(_kernel(2), xs, "var")
    assert out.shape == (3,)
    (_, ndim, xv, ns, _), = s.solver._lib.calls
    assert ndim == 2 and ns == 3 and xv == [0.0, 1.0, 2.0, 3.0, 4.0, 5.0]


def test_predictive_without_test_points():
    s = _solver()
    assert s.predictive(_kernel(), np.zeros((0, 1)), "var").shape == (0,)
    assert s.predictive(_kernel(), np.zeros((0, 1)), "cov").shape == (0, 0)
