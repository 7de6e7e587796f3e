# -*- coding: utf-8 -*-
"""GP.sample_conditional / GP.sample with a caller's generator, on the host: every argument check raises before any
device call, size == 0 returns empty draws, and the rng=None route is still the reference's (predict's mean and
covariance into multivariate_gaussian_samples, numpy's global generator)."""
import numpy as np
import pytest


def _dense_gp():
    import george_b200 as george
    from george_b200 import kernels
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0))
    gp._x = np.linspace(0, 1, 5)[:, None]  # what compute() would leave, without touching the device
    gp._yerr2 = np.zeros(5)
    return gp


class _NoDevice(object):
    """A solver stand-in whose every use fails the test: the checks must raise before the GP reaches it."""

    def __getattr__(self, name):
        raise AssertionError("the solver was used ({0}) before the argument checks finished".format(name))


def _guarded_gp(monkeypatch):
    gp = _dense_gp()
    gp.solver = _NoDevice()

    def no_recompute(*args, **kwargs):
        raise AssertionError("recompute ran before the argument checks finished")

    monkeypatch.setattr(gp, "recompute", no_recompute)
    monkeypatch.setattr(gp, "get_matrix", no_recompute)
    return gp


def test_argument_checks_run_before_any_device_call(monkeypatch):
    gp = _guarded_gp(monkeypatch)
    g = np.random.default_rng(0)
    y, t = np.zeros(5), np.linspace(0, 1, 3)
    with pytest.raises(ValueError, match="jitter applies only"):
        gp.sample_conditional(y, t, jitter=1e-9)
    for bad in (-1e-9, np.nan, np.inf):
        with pytest.raises(ValueError, match="jitter must be finite"):
            gp.sample_conditional(y, t, rng=g, jitter=bad)
    for bad in (0, np.random.PCG64(0), "seed", np.random):
        with pytest.raises(TypeError, match="rng must be"):
            gp.sample_conditional(y, t, rng=bad)
        with pytest.raises(TypeError, match="rng must be"):
            gp.sample(t, rng=bad)
        with pytest.raises(TypeError, match="rng must be"):
            gp.sample(rng=bad)
    with pytest.raises(ValueError, match="size must be"):
        gp.sample_conditional(y, t, -1, rng=g)
    with pytest.raises(ValueError, match="size must be"):
        gp.sample(t, -1, rng=g)
    with pytest.raises(ValueError, match="size must be"):
        gp.sample(size=-2, rng=g)
    with pytest.raises(ValueError, match="Dimension mismatch"):
        gp.sample_conditional(np.zeros(4), t, rng=g)             # y's length
    with pytest.raises(ValueError, match="Dimension mismatch"):
        gp.sample_conditional(y, np.zeros((3, 2)), rng=g)        # t's dimension
    with pytest.raises(ValueError, match="Dimension mismatch"):
        gp.sample(np.zeros((3, 2)), rng=g)


def test_rng_is_not_advanced_by_a_failed_check(monkeypatch):
    gp = _guarded_gp(monkeypatch)
    g = np.random.default_rng(3)
    state = g.bit_generator.state
    with pytest.raises(ValueError):
        gp.sample_conditional(np.zeros(4), np.zeros(3), rng=g)
    with pytest.raises(ValueError):
        gp.sample_conditional(np.zeros(5), np.zeros(3), rng=g, jitter=-1.0)
    assert g.bit_generator.state == state


def test_uncomputed_gp_raises_before_drawing():
    import george_b200 as george
    from george_b200 import kernels
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0))
    g = np.random.default_rng(0)
    state = g.bit_generator.state
    with pytest.raises(RuntimeError, match="You need to compute the model first"):
        gp.sample_conditional(np.zeros(3), np.zeros(4), rng=g)
    with pytest.raises(RuntimeError, match="You need to compute the model first"):
        gp.sample(rng=g)
    assert g.bit_generator.state == state


@pytest.mark.parametrize("make_rng", [lambda: np.random.default_rng(5), lambda: np.random.RandomState(5)])
def test_size_zero_shapes(monkeypatch, make_rng):
    gp = _guarded_gp(monkeypatch)
    for ns in (0, 3):
        t = np.linspace(0, 1, ns)
        g = make_rng()
        out = gp.sample_conditional(np.zeros(5), t, 0, rng=g)
        assert isinstance(out, np.ndarray) and out.shape == (0, ns) and out.dtype == np.float64
        out = gp.sample(t, 0, rng=g)
        assert out.shape == (0, ns)


def test_rng_none_route_is_the_references(monkeypatch):
    """rng=None: predict's (mu, cov) go to multivariate_gaussian_samples, and the draws are numpy's under
    np.random.seed, bit for bit."""
    import george_b200.gp as gpmod
    gp = _dense_gp()
    rng = np.random.default_rng(1)
    a = rng.standard_normal((4, 4))
    mu, cov = rng.standard_normal(4), a @ a.T + np.eye(4)
    calls = []

    def fake_predict(y, t, **kwargs):
        calls.append(kwargs)
        return mu.copy(), cov.copy()

    seen = []
    real = gpmod.multivariate_gaussian_samples

    def spy(matrix, N, mean=None):
        seen.append((np.array(matrix), N, np.array(mean)))
        return real(matrix, N, mean=mean)

    monkeypatch.setattr(gp, "predict", fake_predict)
    monkeypatch.setattr(gpmod, "multivariate_gaussian_samples", spy)
    for size in (1, 3):
        np.random.seed(42)
        got = gp.sample_conditional(np.zeros(5), np.linspace(0, 1, 4), size)
        np.random.seed(42)
        want = np.random.multivariate_normal(mu, cov, size)
        assert np.array_equal(got, want[0] if size == 1 else want)
        m, n, mean = seen[-1]
        assert n == size and np.array_equal(m, cov) and np.array_equal(mean, mu)
    assert calls == [{}, {}]  # predict(y, t): return_cov defaults to True


def test_device_sample_without_device_raises():
    """No CPU fallback: with valid arguments and no H100 the device route raises BGPError, after drawing z once."""
    from george_b200 import _lib
    from george_b200.utils import device_gaussian_samples
    if _lib.load().bgp_device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(_lib.BGPError):
        device_gaussian_samples(np.eye(3), np.zeros((2, 3)), np.zeros(3), 0.0)
    with pytest.raises(ValueError):
        device_gaussian_samples(np.eye(3), np.zeros((2, 4)), np.zeros(3), 0.0)
    import george_b200 as george
    from george_b200 import kernels
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0))
    g = np.random.default_rng(0)
    ref = np.random.default_rng(0)
    with pytest.raises(_lib.BGPError):
        gp.sample(np.linspace(0, 1, 3), 2, rng=g)
    ref.standard_normal((2, 3))
    assert g.bit_generator.state == ref.bit_generator.state


def test_threshold_mirrors_the_header():
    import os
    import re
    from george_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = open(os.path.join(root, "include", "bgp.h")).read()
    m = re.search(r"#define BGP_SAMPLE_DMMA_ROWS (\d+)", src)
    assert m and int(m.group(1)) == _lib.BGP_SAMPLE_DMMA_ROWS
