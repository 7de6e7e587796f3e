# -*- coding: utf-8 -*-
"""GP.batch_sample_conditional on the host: the argument checks that run before the generator or the device is
touched, the empty results and how far they advance the generator, the error raised without a device, and the
per-vector loop taken by solvers without a batched path and by rng=None."""
import numpy as np
import pytest


def _dense_gp(solver=None):
    import george_b200 as george
    from george_b200 import kernels
    kw = {} if solver is None else dict(solver=solver)
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0), mean=0.5, fit_mean=True, **kw)
    gp._x = np.linspace(0, 1, 5)[:, None]  # what compute() would leave, without touching the device
    gp._yerr2 = np.zeros(5)
    return gp


def _rngs():
    return [np.random.default_rng(7), np.random.RandomState(7)]


def _state_of(rng):
    return rng.bit_generator.state if isinstance(rng, np.random.Generator) else rng.get_state()


def _same_state(a, b):
    if isinstance(a, dict):
        return a == b
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


@pytest.mark.parametrize("which", [0, 1])
def test_argument_checks_run_before_the_generator_and_the_device(which):
    import george_b200 as george
    from george_b200 import kernels
    gp = _dense_gp()
    v, y, t = np.zeros((2, len(gp))), np.zeros(5), np.zeros(4)
    bad = [
        (TypeError, "rng must be", lambda g: gp.batch_sample_conditional(v, y, t, rng=object())),
        (ValueError, "jitter must be", lambda g: gp.batch_sample_conditional(v, y, t, rng=g, jitter=-1.0)),
        (ValueError, "jitter must be", lambda g: gp.batch_sample_conditional(v, y, t, rng=g, jitter=np.nan)),
        (ValueError, "size must be", lambda g: gp.batch_sample_conditional(v, y, t, -1, rng=g)),
        (ValueError, "vectors must have shape", lambda g: gp.batch_sample_conditional(v[0], y, t, rng=g)),
        (ValueError, "vectors must have shape",
         lambda g: gp.batch_sample_conditional(np.zeros((2, len(gp) + 1)), y, t, rng=g)),
        (ValueError, "Dimension mismatch", lambda g: gp.batch_sample_conditional(v, np.zeros(4), t, rng=g)),
        (ValueError, "Dimension mismatch", lambda g: gp.batch_sample_conditional(v, y, np.zeros((4, 2)), rng=g)),
        (ValueError, "jitter applies only", lambda g: gp.batch_sample_conditional(v, y, t, jitter=1e-6)),
    ]
    for exc, match, call in bad:
        g = _rngs()[which]
        before = _state_of(g)
        with pytest.raises(exc, match=match):
            call(g)
        assert _same_state(before, _state_of(g)), match
    fresh = george.GP(1.0 * kernels.ExpSquaredKernel(1.0))
    g = _rngs()[which]
    before = _state_of(g)
    with pytest.raises(RuntimeError, match="You need to compute the model first"):
        fresh.batch_sample_conditional(np.zeros((2, len(fresh))), y, t, rng=g)
    assert _same_state(before, _state_of(g))


@pytest.mark.parametrize("which", [0, 1])
@pytest.mark.parametrize("size", [0, 1, 3])
def test_empty_shapes_advance_the_generator_as_the_loop(which, size):
    gp = _dense_gp()
    for nb, ns in ((0, 7), (3, 0), (0, 0), (2, 4)):
        if ns and nb and size:
            continue  # not empty
        g, twin = _rngs()[which], _rngs()[which]
        got = gp.batch_sample_conditional(np.zeros((nb, len(gp))), np.zeros(5), np.zeros(ns), size, rng=g)
        assert got.shape == ((nb, ns) if size == 1 else (nb, size, ns)), (nb, ns, size, got.shape)
        for _ in range(nb):  # the loop's one standard_normal((size, ns)) per member
            twin.standard_normal((size, ns))
        assert _same_state(_state_of(twin), _state_of(g)), (nb, ns, size)
        assert twin.standard_normal() == g.standard_normal()


def test_device_path_without_device_raises():
    """No CPU fallback: with valid arguments and no H100, the batched dense path raises BGPError."""
    import george_b200 as george
    from george_b200 import _lib, kernels
    from george_b200._spec import flatten
    if _lib.load().bgp_device_count() > 0:
        pytest.skip("a GPU is present")
    k = 1.0 * kernels.ExpSquaredKernel(1.0)
    with pytest.raises(_lib.BGPError):
        george.BasicSolver.batch_sample(flatten(k), np.zeros((2, len(k))), np.linspace(0, 1, 5), np.ones((2, 5)),
                                        np.ones((2, 5)), np.linspace(0, 1, 3), np.zeros((2, 3)),
                                        np.zeros((2, 4, 3)), 1e-6)
    with pytest.raises(ValueError, match="mean_add must have shape"):
        george.BasicSolver.batch_sample(flatten(k), np.zeros((2, len(k))), np.linspace(0, 1, 5), np.ones((2, 5)),
                                        np.ones((2, 5)), np.linspace(0, 1, 3), np.zeros((2, 4)),
                                        np.zeros((2, 4, 3)), 1e-6)
    draws, info, draw_info = george.BasicSolver.batch_sample(
        flatten(k), np.zeros((0, len(k))), np.linspace(0, 1, 5), np.ones((0, 5)), np.ones((0, 5)),
        np.linspace(0, 1, 3), np.zeros((0, 3)), np.zeros((0, 4, 3)), 1e-6)
    assert draws.shape == (0, 4, 3) and info.shape == (0,) and draw_info.shape == (0,)
    gp = _dense_gp()
    with pytest.raises(_lib.BGPError):
        gp.batch_sample_conditional(np.zeros((2, len(gp))), np.zeros(5), np.linspace(0, 1, 3),
                                    rng=np.random.default_rng(0))
    assert george.HODLRSolver.batch_sample is None
    assert getattr(george.TrivialSolver, "batch_sample", None) is None


def _spy(monkeypatch):
    """Replace GP.sample_conditional by a host stand-in that records its calls and returns the first parameter."""
    import george_b200 as george
    calls = []

    def fake(self, y, t, size=1, *, rng=None, jitter=None):
        calls.append((self.get_parameter_vector().copy(), rng, jitter, size))
        self.kernel.dirty = True  # as a refactorisation would leave it changed
        ns = len(np.atleast_1d(t))
        v = self.get_parameter_vector()[0] + (rng.standard_normal((size, ns)) if rng is not None else 0.0)
        out = np.broadcast_to(v, (size, ns)).copy()
        return out[0] if size == 1 else out

    monkeypatch.setattr(george.GP, "sample_conditional", fake)
    return calls


def _check_loop(gp, monkeypatch, rng, size, jitter):
    calls = _spy(monkeypatch)
    vecs = gp.get_parameter_vector() + np.arange(3.0)[:, None] * np.ones(len(gp))
    before = (gp.get_parameter_vector(include_frozen=True).copy(), [m.dirty for m in gp.models.values()],
              gp.solver, gp._alpha)
    got = gp.batch_sample_conditional(vecs, np.zeros(5), np.linspace(0, 1, 4), size, rng=rng, jitter=jitter)
    assert [c[1] for c in calls] == [rng] * 3 and [c[2] for c in calls] == [jitter] * 3
    for b, c in enumerate(calls):
        assert np.array_equal(c[0], vecs[b])
    assert got.shape == ((3, 4) if size == 1 else (3, size, 4))
    if rng is None:
        assert np.array_equal(got[..., 0].reshape(3, -1)[:, 0], vecs[:, 0])
    assert np.array_equal(gp.get_parameter_vector(include_frozen=True), before[0])
    assert [m.dirty for m in gp.models.values()] == before[1]
    assert gp.solver is before[2] and gp._alpha is before[3]


@pytest.mark.parametrize("size", [1, 3])
def test_rng_none_runs_the_loop_and_restores_the_gp(monkeypatch, size):
    _check_loop(_dense_gp(), monkeypatch, None, size, None)


@pytest.mark.parametrize("size", [1, 3])
def test_solver_without_the_hook_runs_the_loop_and_restores_the_gp(monkeypatch, size):
    import george_b200 as george

    class NoBatch(george.BasicSolver):
        batch_sample = None

    for solver in (NoBatch, george.HODLRSolver):
        g = np.random.default_rng(3)
        _check_loop(_dense_gp(solver), monkeypatch, g, size, 1e-6)
