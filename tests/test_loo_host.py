# -*- coding: utf-8 -*-
"""Leave-one-out cross-validation on the host (no GPU): ``GP.loo_predict``, ``GP.loo_log_likelihood`` and
``GP.grad_loo_log_likelihood``.

* ``TrivialSolver`` (host route: K^-1 from ``apply_inverse``) against a brute-force refit of N - 1 points, with a fitted
  non-constant white-noise model and a fitted mean model, and the gradient against centred differences;
* the argument and ``quiet`` semantics, the gradient layout, frozen parameters and ``return_value``, with a stub solver
  whose ``loo_terms`` hook returns fixed arrays;
* ``ShardedHODLRSolver.loo_terms`` raises ``NotImplementedError`` on every rank of a gloo world of two before any
  collective.
"""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

N = 12


class _LineMean(object):
    """mean(x) = m * x + b, a fitted mean model with a gradient (modeling protocol)."""

    def __new__(cls, m, b):
        from george_b200.modeling import Model

        class LineMean(Model):
            parameter_names = ("m", "b")

            def get_value(self, x):
                return self.m * np.asarray(x).flatten() + self.b

            def compute_gradient(self, x):
                x = np.asarray(x).flatten()
                return np.vstack([x, np.ones_like(x)])

        return LineMean(m=m, b=b)


class _LogLinearNoise(object):
    """white noise log-variance wn(x) = a + s * x: a fitted non-constant white-noise model."""

    def __new__(cls, a, s):
        from george_b200.modeling import Model

        class LogLinearNoise(Model):
            parameter_names = ("a", "s")

            def get_value(self, x):
                return self.a + self.s * np.asarray(x).flatten()

            def compute_gradient(self, x):
                x = np.asarray(x).flatten()
                return np.vstack([np.ones_like(x), x])

        return LogLinearNoise(a=a, s=s)


def _data(n=N, seed=3):
    rng = np.random.default_rng(seed)
    x = np.sort(rng.uniform(0, 5, n))
    yerr = 0.2 + 0.1 * rng.random(n)
    y = 0.4 * x - 0.3 + 0.5 * rng.standard_normal(n)
    return x, yerr, y


def _trivial_gp():
    import george_b200 as george
    x, yerr, y = _data()
    gp = george.GP(mean=_LineMean(0.3, -0.1), fit_mean=True, white_noise=_LogLinearNoise(-2.0, 0.1),
                   fit_white_noise=True)
    gp.compute(x, yerr)
    return gp, x, yerr, y


def _brute(gp, x, yerr, y):
    """(mu, var, value) of the N - 1 refits: the covariance is diagonal, so y_i given the others is N(mean_i, var_i)
    with var_i = yerr_i^2 + exp(wn(x_i)); written as the general conditional to check the formulas, not the shortcut."""
    mean = gp.mean.get_value(x)
    K = np.diag(yerr ** 2 + np.exp(gp.white_noise.get_value(x)))
    n = len(x)
    mu, var = np.empty(n), np.empty(n)
    for i in range(n):
        k = np.delete(np.arange(n), i)
        w = np.linalg.solve(K[np.ix_(k, k)], K[k, i])
        mu[i] = mean[i] + w @ (y[k] - mean[k])
        var[i] = K[i, i] - K[i, k] @ w
    value = np.sum(-0.5 * np.log(2 * np.pi * var) - 0.5 * (y - mu) ** 2 / var)
    return mu, var, value


def test_trivial_against_brute_force_refit():
    gp, x, yerr, y = _trivial_gp()
    mu, var = gp.loo_predict(y)
    mu_ref, var_ref, value_ref = _brute(gp, x, yerr, y)
    assert np.allclose(mu, mu_ref, rtol=1e-13, atol=1e-13)
    assert np.allclose(var, var_ref, rtol=1e-13)
    assert abs(gp.loo_log_likelihood(y) - value_ref) <= 1e-12 * abs(value_ref)


def test_trivial_gradient_against_centred_differences():
    gp, x, yerr, y = _trivial_gp()
    v0 = gp.get_parameter_vector()
    value, grad = gp.grad_loo_log_likelihood(y, return_value=True)
    assert value == gp.loo_log_likelihood(y)
    assert grad.shape == (len(gp),) == (4,)  # mean (m, b), white noise (a, s); EmptyKernel has no parameters
    h = 1e-6
    fd = np.empty(len(v0))
    for k in range(len(v0)):
        e = np.zeros(len(v0))
        e[k] = h
        gp.set_parameter_vector(v0 + e)
        vp = _brute(gp, x, yerr, y)[2]
        gp.set_parameter_vector(v0 - e)
        vm = _brute(gp, x, yerr, y)[2]
        fd[k] = (vp - vm) / (2 * h)
    gp.set_parameter_vector(v0)
    assert np.allclose(grad, fd, rtol=1e-7, atol=1e-7), (grad, fd)


# ---- a stub solver: the GP layer around fixed loo_terms ------------------------------------------------------------

ALPHA = np.linspace(-1.0, 1.0, N)
D = np.linspace(1.0, 2.0, N)
BETA = np.linspace(0.5, -0.5, N)
DIAG_A = np.linspace(-0.2, 0.3, N)


class _StubSolver(object):
    """Records loo_terms calls and returns fixed arrays; g[p] = 10 p + 1 over ALL kernel parameters (zeros where
    ``which`` is 0)."""

    calls = []
    d = D

    def __init__(self, kernel, **kwargs):
        self.kernel = kernel
        self.computed = False

    def compute(self, x, yerr):
        self.log_determinant = 0.0
        self.computed = True

    def apply_inverse(self, y, in_place=False):
        raise AssertionError("the hook route must not form K^-1")

    def dot_solve(self, y):
        return 0.0

    def loo_terms(self, r, which=None):
        _StubSolver.calls.append((np.array(r), None if which is None else np.array(which)))
        if which is None:
            return ALPHA.copy(), self.d.copy()
        g = (10.0 * np.arange(len(which)) + 1.0) * (np.asarray(which) != 0)
        return ALPHA.copy(), self.d.copy(), BETA.copy(), g, DIAG_A.copy()


def _stub_gp(freeze=()):
    import george_b200 as george
    from george_b200 import kernels
    kernel = 2.0 * kernels.ExpSquaredKernel(1.5)  # parameters: k1:log_constant, k2:metric:log_M_0_0
    gp = george.GP(kernel, mean=_LineMean(0.3, -0.1), fit_mean=True, white_noise=_LogLinearNoise(-2.0, 0.1),
                   fit_white_noise=True, solver=_StubSolver)
    for name in freeze:
        gp.freeze_parameter(name)
    x, yerr, _ = _data()
    gp.compute(x, yerr)
    _StubSolver.calls = []
    _StubSolver.d = D
    return gp, x


def _value(alpha, d):
    return np.sum(-0.5 * np.log(2 * np.pi) + 0.5 * np.log(d) - alpha ** 2 / (2 * d))


def test_stub_value_and_predict():
    gp, x = _stub_gp()
    y = np.arange(N, dtype=np.float64)
    mu, var = gp.loo_predict(y)
    assert np.array_equal(mu, y - ALPHA / D) and np.array_equal(var, 1.0 / D)
    assert gp.loo_log_likelihood(y) == _value(ALPHA, D)
    r, which = _StubSolver.calls[0]
    assert which is None and np.array_equal(r, y - gp.mean.get_value(x))


def test_stub_gradient_layout():
    gp, x = _stub_gp()
    y = np.zeros(N)
    grad = gp.grad_loo_log_likelihood(y)
    r, which = _StubSolver.calls[-1]
    assert np.array_equal(which, [1, 1])
    wn = gp.white_noise.get_value(x)
    ref = np.concatenate([
        [np.dot(x, BETA), np.sum(BETA)],                                       # mean: dmu . beta
        [np.sum(np.exp(wn) * DIAG_A), np.sum(np.exp(wn) * DIAG_A * x)],        # white noise: A_ii exp(wn) dwn
        [1.0, 11.0],                                                           # kernel: g as given, no factor 1/2
    ])
    assert np.allclose(grad, ref, rtol=1e-14, atol=1e-14)
    assert len(grad) == len(gp) == 6


def test_stub_frozen_parameters():
    gp, x = _stub_gp(freeze=("kernel:k1:log_constant", "mean:b", "white_noise:s"))
    grad = gp.grad_loo_log_likelihood(np.zeros(N))
    _, which = _StubSolver.calls[-1]
    assert np.array_equal(which, [0, 1])  # which covers every kernel parameter
    wn = gp.white_noise.get_value(x)
    assert np.allclose(grad, [np.dot(x, BETA), np.sum(np.exp(wn) * DIAG_A), 11.0], rtol=1e-14, atol=1e-14)


def test_stub_return_value_is_the_value():
    gp, _ = _stub_gp()
    y = np.ones(N)
    value, grad = gp.grad_loo_log_likelihood(y, return_value=True)
    assert value == gp.loo_log_likelihood(y)
    assert np.array_equal(grad, gp.grad_loo_log_likelihood(y))


@pytest.mark.parametrize("bad", [0.0, -1.0, np.nan, np.inf])
def test_stub_nonpositive_d_gives_minus_inf(bad):
    gp, _ = _stub_gp()
    d = D.copy()
    d[4] = bad
    _StubSolver.d = d
    assert gp.loo_log_likelihood(np.zeros(N)) == -np.inf


def test_nan_mean():
    gp, _ = _stub_gp()
    gp.set_parameter("mean:b", np.nan)
    y = np.zeros(N)
    assert gp.loo_log_likelihood(y, quiet=True) == -np.inf
    with pytest.raises(ValueError, match="mean function"):
        gp.loo_log_likelihood(y)
    assert np.array_equal(gp.grad_loo_log_likelihood(y, quiet=True), np.zeros(len(gp)))
    value, grad = gp.grad_loo_log_likelihood(y, quiet=True, return_value=True)
    assert value == -np.inf and np.array_equal(grad, np.zeros(len(gp)))
    with pytest.raises(ValueError, match="mean function"):
        gp.grad_loo_log_likelihood(y)
    with pytest.raises(ValueError, match="mean function"):
        gp.loo_predict(y)
    assert _StubSolver.calls == []


def test_dimension_mismatch():
    gp, _ = _stub_gp()
    for fn in (gp.loo_predict, gp.loo_log_likelihood, gp.grad_loo_log_likelihood):
        with pytest.raises(ValueError, match="Dimension mismatch"):
            fn(np.zeros(N + 1))


def test_before_compute():
    import george_b200 as george
    gp = george.GP(solver=_StubSolver)
    for fn in (gp.loo_predict, gp.loo_log_likelihood, gp.grad_loo_log_likelihood):
        with pytest.raises(RuntimeError, match="compute"):
            fn(np.zeros(N))


def test_host_route_nonpositive_d_names_the_point():
    """The host route checks d before the gradient, as the device route does; quiet absorbs it."""
    import george_b200 as george

    class Negative(george.solvers.TrivialSolver):
        def apply_inverse(self, y, in_place=False):
            y = np.array(y, dtype=np.float64)
            y[3] *= -1.0
            return y

    x, yerr, y = _data()
    gp = george.GP(solver=Negative)
    gp.compute(x, yerr)
    assert gp.loo_log_likelihood(y) == -np.inf
    with pytest.raises(ValueError, match="point 3"):
        gp.grad_loo_log_likelihood(y)
    assert np.array_equal(gp.grad_loo_log_likelihood(y, quiet=True), np.zeros(len(gp)))


# ---- ShardedHODLRSolver: NotImplementedError on every rank, before any collective -----------------------------------

def _sharded_worker(rank, world, port, tmp):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    from george_b200 import kernels
    from george_b200.parallel import ShardedHODLRSolver
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    s = ShardedHODLRSolver(1.0 * kernels.ExpKernel(1.0))
    s._n, s._computed = N, True  # no native handle: loo_terms must not reach one
    raised = []
    for which in (None, np.ones(2, dtype=np.uint32)):
        try:
            s.loo_terms(np.zeros(N), which)
        except NotImplementedError as exc:
            raised.append("ShardedHODLRSolver" in str(exc))
    # both ranks get here: nothing above waited on a collective
    flag = torch.tensor([1.0], dtype=torch.float64)
    dist.all_reduce(flag)
    np.save(os.path.join(tmp, "ok{0}.npy".format(rank)), np.array([raised == [True, True] and flag.item() == world]))
    dist.destroy_process_group()


def test_sharded_loo_not_implemented_gloo_world2(tmp_path):
    import torch.multiprocessing as mp
    port = 29500 + (os.getpid() % 2000) + 3
    mp.spawn(_sharded_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    for r in range(2):
        assert np.load(os.path.join(str(tmp_path), "ok{0}.npy".format(r)))[0]
