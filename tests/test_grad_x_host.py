# -*- coding: utf-8 -*-
"""``GP.grad_log_likelihood_x`` on the host (no GPU), around a stub solver whose ``grad_terms`` / ``grad_x_terms`` hooks
return fixed arrays: the output layout, ``return_gradient`` against ``grad_log_likelihood``, ``quiet``, the model and
dimension checks (raised before the solver is reached), frozen parameters and the GP's state.  Then
``ShardedHODLRSolver.grad_x_terms``: its buffers, and its argument errors on every rank of a gloo world of two with no
rank left waiting.  The device arithmetic is tested in tests/test_gpu_grad_x.py."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
from numpy.linalg import LinAlgError

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

N = 10


class _Stub(object):
    """A solver plug-in with K^-1 = 2 I: alpha = 2 r, g[p] = (p + 1) * sum(r) where which[p], diagA = alpha^2 - 2 and
    dx[i, q] = 10 i + q + sum(r).  ``fail`` makes the hooks raise ValueError; every hook call is recorded in ``calls``."""
    calls = []
    fail = False
    fail_compute = False

    def __init__(self, kernel):
        self.kernel = kernel
        self.computed = False
        self.log_determinant = None

    def compute(self, x, yerr):
        if _Stub.fail_compute:
            raise LinAlgError("not positive definite")
        self._x = np.asarray(x)
        self.log_determinant = -len(x) * np.log(2.0)
        self.computed = True

    def apply_inverse(self, y, in_place=False):
        return 2.0 * np.asarray(y, dtype=np.float64)

    def dot_solve(self, y):
        return 2.0 * float(np.dot(y, y))

    def get_inverse(self):
        return 2.0 * np.eye(len(self._x))

    def _terms(self, r, which):
        if _Stub.fail:
            raise ValueError("stub failure")
        alpha = 2.0 * r
        g = np.zeros(0) if which is None else np.array([(p + 1) * r.sum() if w else 0.0 for p, w in enumerate(which)])
        return alpha, g, alpha ** 2 - 2.0

    def grad_terms(self, r, which):
        _Stub.calls.append(("grad_terms", None if which is None else list(which)))
        return self._terms(r, which)

    def grad_x_terms(self, r, which):
        _Stub.calls.append(("grad_x_terms", None if which is None else list(which)))
        alpha, g, diag = self._terms(r, which)
        n, nd = self._x.shape
        dx = 10.0 * np.arange(n)[:, None] + np.arange(nd)[None, :] + r.sum()
        return alpha, g, diag, dx


@pytest.fixture(autouse=True)
def _reset():
    _Stub.calls, _Stub.fail, _Stub.fail_compute = [], False, False
    yield


def _data(nd=1, seed=5):
    rng = np.random.default_rng(seed)
    x = rng.uniform(0, 3, (N, nd))
    return (x[:, 0] if nd == 1 else x), 0.1 + 0.05 * rng.random(N), rng.standard_normal(N)


def _gp(nd=1, **kwargs):
    import george_b200 as george
    from george_b200 import kernels
    k = 1.3 * kernels.ExpSquaredKernel(0.7, ndim=nd) if nd > 1 else 1.3 * kernels.ExpSquaredKernel(0.7)
    gp = george.GP(k, solver=_Stub, **kwargs)
    x, yerr, y = _data(nd)
    gp.compute(x, yerr)
    return gp, x, y


@pytest.mark.parametrize("nd", [1, 3])
def test_layout_and_shape(nd):
    gp, x, y = _gp(nd)
    dx = gp.grad_log_likelihood_x(y)
    assert dx.shape == (N, nd) and dx.dtype == np.float64
    r = y - 0.0
    assert np.array_equal(dx, 10.0 * np.arange(N)[:, None] + np.arange(nd)[None, :] + r.sum())
    # without return_gradient the parameter contraction is skipped
    assert _Stub.calls == [("grad_x_terms", None)]


@pytest.mark.parametrize("kwargs", [
    dict(),
    dict(mean=0.4, fit_mean=True),
    dict(mean=0.4, fit_mean=True, white_noise=-3.0, fit_white_noise=True),
    dict(white_noise=-3.0, fit_white_noise=True, fit_kernel=False),
    dict(mean=0.4, fit_mean=True, fit_kernel=False),
])
def test_return_gradient_is_grad_log_likelihood(kwargs):
    gp, x, y = _gp(**kwargs)
    grad, dx = gp.grad_log_likelihood_x(y, return_gradient=True)
    ref = gp.grad_log_likelihood(y)
    assert grad.shape == ref.shape == (len(gp),)
    assert np.array_equal(grad, ref)
    assert np.array_equal(dx, gp.grad_log_likelihood_x(y))


def test_frozen_parameters():
    gp, x, y = _gp(mean=0.4, fit_mean=True)
    gp.freeze_parameter("kernel:k1:log_constant")
    mask = gp.kernel.unfrozen_mask
    assert not mask.all()
    grad, dx = gp.grad_log_likelihood_x(y, return_gradient=True)
    assert np.array_equal(grad, gp.grad_log_likelihood(y))
    assert len(grad) == len(gp) == 1 + int(mask.sum())
    assert _Stub.calls[0] == ("grad_x_terms", [int(m) for m in mask])


def test_quiet_absorbs_a_failure():
    gp, x, y = _gp(mean=0.4, fit_mean=True)
    _Stub.fail = True
    with pytest.raises(ValueError, match="stub failure"):
        gp.grad_log_likelihood_x(y)
    dx = gp.grad_log_likelihood_x(y, quiet=True)
    assert dx.shape == (N, 1) and not dx.any()
    grad, dx = gp.grad_log_likelihood_x(y, quiet=True, return_gradient=True)
    assert grad.shape == (len(gp),) and not grad.any() and not dx.any()


def test_quiet_absorbs_a_failed_factorisation():
    gp, x, y = _gp()
    gp.set_parameter_vector(gp.get_parameter_vector() + 0.1)  # dirty: the next call refactorises
    _Stub.fail_compute = True
    grad, dx = gp.grad_log_likelihood_x(y, quiet=True, return_gradient=True)
    assert not grad.any() and not dx.any() and dx.shape == (N, 1)
    with pytest.raises(LinAlgError):
        gp.grad_log_likelihood_x(y)


def _line_model():
    from george_b200.modeling import Model

    class Line(Model):
        parameter_names = ("m", "b")

        def get_value(self, x):
            return self.m * np.asarray(x).flatten() + self.b

    return Line(m=0.1, b=-1.0)


def test_non_constant_mean_raises_before_the_solver():
    gp, x, y = _gp(mean=_line_model())
    _Stub.calls = []
    with pytest.raises(NotImplementedError, match="constant mean"):
        gp.grad_log_likelihood_x(y)
    assert _Stub.calls == []


def test_non_constant_white_noise_raises_before_the_solver():
    gp, x, y = _gp(white_noise=_line_model())
    _Stub.calls = []
    with pytest.raises(NotImplementedError, match="constant white-noise"):
        gp.grad_log_likelihood_x(y, return_gradient=True)
    assert _Stub.calls == []


def test_more_than_eight_dimensions_raise_before_the_solver():
    gp, x, y = _gp(nd=9)
    _Stub.calls = []
    gp.set_parameter_vector(gp.get_parameter_vector())  # dirty: a refactorisation would be device work
    computed = gp.computed
    with pytest.raises(ValueError, match="at most 8 dimensions"):
        gp.grad_log_likelihood_x(y)
    assert _Stub.calls == [] and gp.computed == computed


def test_state_unchanged():
    gp, x, y = _gp(mean=0.4, fit_mean=True)
    gp.log_likelihood(y)
    alpha, cached_y, p = gp._alpha, gp._y, gp.get_parameter_vector()
    gp.grad_log_likelihood_x(y, return_gradient=True)
    assert gp._alpha is alpha and gp._y is cached_y and gp.computed
    assert np.array_equal(gp.get_parameter_vector(), p)


# ---- ShardedHODLRSolver.grad_x_terms ---------------------------------------------------------------------------------

class _FakeLib(object):
    """bgp_hodlr_grad_x_terms: records (which, r) and writes alpha = 2 r, g[p] = 10 + p where which[p], diag = -r and
    dx[i, q] = i + 0.5 q."""

    def __init__(self, n, npar, nd):
        self.n, self.npar, self.nd, self.calls = n, npar, nd, []

    def bgp_hodlr_grad_x_terms(self, ptr, which, r, alpha, g, diag, dx):
        dp = C.POINTER(C.c_double)
        rv = [C.cast(r, dp)[i] for i in range(self.n)]
        wv = None if which is None else [C.cast(which, C.POINTER(C.c_uint32))[p] for p in range(self.npar)]
        self.calls.append((ptr, wv, rv))
        a, d, x = C.cast(alpha, dp), C.cast(diag, dp), C.cast(dx, dp)
        for i in range(self.n):
            a[i], d[i] = 2.0 * rv[i], -rv[i]
            for q in range(self.nd):
                x[i * self.nd + q] = i + 0.5 * q
        if wv is not None:
            gg = C.cast(g, dp)
            for p in range(self.npar):
                gg[p] = 10.0 + p if wv[p] else 0.0
        return 0


class _FakeNative(object):
    def __init__(self, n, npar, nd):
        self._lib = _FakeLib(n, npar, nd)
        self._ptr = C.c_void_p(1234)
        self._ndim = nd


def _sharded(n=6, npar=3, nd=2, computed=True):
    from george_b200 import kernels
    from george_b200.parallel import ShardedHODLRSolver
    s = ShardedHODLRSolver(1.0 * kernels.ExpKernel(1.0))
    if computed:
        s.solver = _FakeNative(n, npar, nd)
        s._n = n
        s._computed = True
    return s


def test_sharded_grad_x_terms_buffers():
    s = _sharded(n=6, npar=3, nd=2)
    r = np.arange(6, dtype=np.int64)
    alpha, g, diag, dx = s.grad_x_terms(r, [1, 0, 1])
    assert np.array_equal(alpha, 2.0 * r) and np.array_equal(diag, -1.0 * r) and np.array_equal(g, [10.0, 0.0, 12.0])
    assert dx.shape == (6, 2) and np.array_equal(dx, np.arange(6)[:, None] + 0.5 * np.arange(2)[None, :])
    alpha, g, diag, dx = s.grad_x_terms(r, None)
    assert g.shape == (0,) and s.solver._lib.calls[-1][1] is None


def _sharded_worker(rank, world, port, tmp):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    results = []
    s = _sharded(computed=False)
    try:
        s.grad_x_terms(np.ones(6), np.ones(3, dtype=np.uint32))
    except RuntimeError as exc:
        results.append("compute" in str(exc))
    s = _sharded()
    for r in (np.ones(5), np.ones((6, 1)), np.r_[np.ones(5), np.nan]):
        try:
            s.grad_x_terms(r, np.ones(3, dtype=np.uint32))
        except ValueError:
            results.append(True)
    results.append(s.solver._lib.calls == [])
    # both ranks get here: nothing above waited on a collective
    flag = torch.tensor([1.0], dtype=torch.float64)
    dist.all_reduce(flag)
    np.save(os.path.join(tmp, "ok{0}.npy".format(rank)), np.array([results == [True] * 5 and flag.item() == world]))
    dist.destroy_process_group()


def test_sharded_grad_x_terms_argument_errors_gloo_world2(tmp_path):
    import torch.multiprocessing as mp
    port = 29500 + (os.getpid() % 2000) + 7
    mp.spawn(_sharded_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    for r in range(2):
        assert np.load(os.path.join(str(tmp_path), "ok{0}.npy".format(r)))[0]
