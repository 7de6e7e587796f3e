# -*- coding: utf-8 -*-
"""ShardedHODLRSolver.grad_terms on CPU: its argument checks and the buffers it hands to bgp_hodlr_grad_terms, with the
native handle replaced by a stand-in that records the call and fills the outputs.  The collective arithmetic itself
needs several GPUs (tools/mgpu_check.py); one shard's part runs on one GPU in tests/test_gpu_hodlr_shard_grad.py."""
import ctypes as C

import numpy as np
import pytest


class _FakeLib(object):
    """bgp_hodlr_grad_terms: records (which, r) and writes alpha = 2 r, g[p] = 10 + p where which[p], diag = -r."""

    def __init__(self, n, npar):
        self.n, self.npar, self.calls = n, npar, []

    def bgp_hodlr_grad_terms(self, ptr, which, r, alpha, g, diag):
        dp = C.POINTER(C.c_double)
        w = C.cast(which, C.POINTER(C.c_uint32))
        rv = [C.cast(r, dp)[i] for i in range(self.n)]
        wv = [w[p] for p in range(self.npar)]
        self.calls.append((ptr, wv, rv))
        a, gg, d = C.cast(alpha, dp), C.cast(g, dp), C.cast(diag, dp)
        for i in range(self.n):
            a[i], d[i] = 2.0 * rv[i], -rv[i]
        for p in range(self.npar):
            gg[p] = 10.0 + p if wv[p] else 0.0
        return 0


class _FakeNative(object):
    def __init__(self, n, npar):
        self._lib = _FakeLib(n, npar)
        self._ptr = C.c_void_p(1234)


def _solver(n=6, npar=3, computed=True):
    from george_b200 import kernels
    from george_b200.parallel import ShardedHODLRSolver
    s = ShardedHODLRSolver(1.0 * kernels.ExpKernel(1.0))
    if computed:
        s.solver = _FakeNative(n, npar)
        s._n = n
        s._computed = True
    return s


def test_grad_terms_before_compute_raises():
    with pytest.raises(RuntimeError, match="compute"):
        _solver(computed=False).grad_terms(np.ones(6), np.ones(2, dtype=np.uint32))


@pytest.mark.parametrize("shape", [(5,), (7,), (6, 1), (1, 6)])
def test_grad_terms_rejects_a_misshaped_r(shape):
    s = _solver()
    with pytest.raises(ValueError, match="dimension mismatch"):
        s.grad_terms(np.ones(shape), np.ones(3, dtype=np.uint32))
    assert s.solver._lib.calls == []


def test_grad_terms_shapes_and_buffers():
    """(alpha, g, diag) with BasicSolver.grad_terms' shapes; r and which reach the library as float64 / uint32."""
    s = _solver(n=6, npar=3)
    r = np.arange(6, dtype=np.int64)  # converted to float64
    alpha, g, diag = s.grad_terms(r, [1, 0, 1])
    assert alpha.shape == (6,) and diag.shape == (6,) and g.shape == (3,)
    assert alpha.dtype == g.dtype == diag.dtype == np.float64
    assert np.array_equal(alpha, 2.0 * r) and np.array_equal(diag, -1.0 * r)
    assert np.array_equal(g, [10.0, 0.0, 12.0])
    (ptr, wv, rv), = s.solver._lib.calls
    assert ptr.value == 1234 and wv == [1, 0, 1] and rv == [float(v) for v in r]


def test_grad_terms_without_kernel_parameters():
    s = _solver(n=4, npar=0)
    alpha, g, diag = s.grad_terms(np.ones(4), np.zeros(0, dtype=np.uint32))
    assert g.shape == (0,) and alpha.shape == diag.shape == (4,)
