# -*- coding: utf-8 -*-
"""ShardedHODLRSolver.apply_symmetric_factor and symmetric_log_determinant on CPU: their argument checks, output shapes
and the buffers they hand to bgp_hodlr_sym_apply / bgp_hodlr_sym_log_determinant, with the native handle replaced by a
stand-in that records the call and fills the output.  The collective arithmetic itself needs several GPUs
(tools/mgpu_check.py); the shards' steps run on one GPU in tests/test_gpu_hodlr_shard_sqrt.py."""
import ctypes as C

import numpy as np
import pytest

N = 5


class _FakeLib(object):
    """bgp_hodlr_sym_apply: records (ptr, z as passed, nrhs, ldz, transpose) and writes z <- 10 z + transpose;
    bgp_hodlr_sym_log_determinant writes -3.25."""

    def __init__(self):
        self.calls = []

    def bgp_hodlr_sym_apply(self, ptr, z, nrhs, ldz, transpose):
        p = C.cast(z, C.POINTER(C.c_double))
        self.calls.append((ptr, [p[i] for i in range(nrhs * ldz)], nrhs, ldz, transpose))
        for i in range(nrhs * ldz):
            p[i] = 10.0 * p[i] + transpose
        return 0

    def bgp_hodlr_sym_log_determinant(self, ptr, out):
        self.calls.append((ptr, "logdet"))
        out._obj.value = -3.25
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
        s._n = N
        s._computed = True
    return s


def test_before_compute_raises():
    s = _solver(computed=False)
    with pytest.raises(RuntimeError, match="compute"):
        s.apply_symmetric_factor(np.ones(N))
    with pytest.raises(RuntimeError, match="compute"):
        s.symmetric_log_determinant


@pytest.mark.parametrize("shape", [(N + 1,), (N - 1, 2), (N, 2, 2), ()])
def test_dimension_mismatch(shape):
    s = _solver()
    with pytest.raises(ValueError, match="dimension mismatch"):
        s.apply_symmetric_factor(np.zeros(shape))
    assert s.solver._lib.calls == []


@pytest.mark.parametrize("transpose", [False, True])
def test_vector_keeps_its_shape(transpose):
    s = _solver()
    z = np.arange(N, dtype=np.int64)  # converted to float64
    out = s.apply_symmetric_factor(z, transpose=transpose)
    assert out.dtype == np.float64 and out.shape == (N,)
    assert np.array_equal(out, 10.0 * z + transpose)
    assert np.array_equal(z, np.arange(N))  # the input is not written
    (ptr, buf, nrhs, ldz, tr), = s.solver._lib.calls
    assert ptr.value == 4321 and nrhs == 1 and ldz == N and tr == int(transpose) and buf == list(range(N))


def test_matrix_is_handed_over_column_major():
    s = _solver()
    z = np.arange(3 * N, dtype=np.float64).reshape(N, 3)  # C order: the library sees it column-major
    out = s.apply_symmetric_factor(z)
    assert out.shape == (N, 3) and np.array_equal(out, 10.0 * z)
    (_, buf, nrhs, ldz, tr), = s.solver._lib.calls
    assert nrhs == 3 and ldz == N and tr == 0 and buf == list(z.T.ravel())


def test_symmetric_log_determinant():
    s = _solver()
    assert s.symmetric_log_determinant == -3.25
    (ptr, what), = s.solver._lib.calls
    assert ptr.value == 4321 and what == "logdet"


def test_no_sample_prior_hook():
    """GP.sample on a sharded solver stays apply_sqrt's NotImplementedError: no sample_prior hook."""
    from george_b200.parallel import ShardedHODLRSolver
    assert getattr(ShardedHODLRSolver, "sample_prior", None) is None
    with pytest.raises(NotImplementedError):
        _solver().apply_sqrt(np.ones(N))
