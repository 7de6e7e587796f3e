# -*- coding: utf-8 -*-
"""GP.sample on the HODLR solver's symmetric factor, on the host: the argument checks and the generator's draw come
before any device call, rng=None keeps the reference's route (apply_sqrt, NotImplementedError on HODLR), and without a
GPU the call raises instead of computing anything."""
import numpy as np
import pytest


def _hodlr_gp():
    import george_b200 as george
    from george_b200 import kernels
    gp = george.GP(1.0 * kernels.Matern32Kernel(1.0), solver=george.HODLRSolver, min_size=64, tol=1e-10)
    gp._x = np.linspace(0, 1, 5)[:, None]  # what compute() would leave, without touching the device
    gp._yerr2 = np.zeros(5)
    return gp


class _Recorder(object):
    """A solver stand-in with the HODLR hook: records the z it is handed."""

    def __init__(self):
        self.z = None

    def sample_prior(self, z):
        self.z = z.copy()
        return 2.0 * z

    def apply_sqrt(self, r):
        raise AssertionError("the hook's route must not call apply_sqrt")


def test_checks_and_generator_before_any_device_call(monkeypatch):
    gp = _hodlr_gp()
    calls = []
    monkeypatch.setattr(gp, "recompute", lambda *a, **k: calls.append("recompute") or True)
    for bad in (0, "seed", np.random):
        with pytest.raises(TypeError, match="rng must be"):
            gp.sample(rng=bad)
    with pytest.raises(ValueError, match="size must be"):
        gp.sample(size=-1, rng=np.random.default_rng(0))
    assert calls == []
    rec = _Recorder()
    gp.solver = rec
    g, ref = np.random.default_rng(4), np.random.default_rng(4)
    d = gp.sample(size=3, rng=g)
    z = ref.standard_normal((3, 5))
    assert np.array_equal(rec.z, z)                     # one standard_normal((size, N)), before the solver
    assert np.array_equal(d, 2.0 * z + gp._call_mean(gp._x))
    assert np.array_equal(g.standard_normal(2), ref.standard_normal(2))
    assert calls == ["recompute"]
    assert gp.sample(size=1, rng=np.random.default_rng(4)).shape == (5,)


def test_hook_declining_falls_back_to_apply_sqrt(monkeypatch):
    gp = _hodlr_gp()
    monkeypatch.setattr(gp, "recompute", lambda *a, **k: True)

    class Declines(object):
        def sample_prior(self, z):
            return None

        def apply_sqrt(self, r):
            raise NotImplementedError("apply_sqrt is not implemented for the HODLRSolver")

    gp.solver = Declines()
    with pytest.raises(NotImplementedError):
        gp.sample(size=2, rng=np.random.default_rng(0))


def test_apply_sqrt_and_rng_none_keep_the_reference_route(monkeypatch):
    import george_b200 as george
    from george_b200 import kernels
    h = george.HODLRSolver(kernels.ExpSquaredKernel(1.0))
    with pytest.raises(NotImplementedError):
        h.apply_sqrt(np.zeros(3))
    gp = _hodlr_gp()
    monkeypatch.setattr(gp, "recompute", lambda *a, **k: True)
    rec = _Recorder()
    gp.solver = rec
    with pytest.raises(AssertionError, match="apply_sqrt"):
        gp.sample(size=2)  # rng=None: apply_sqrt, never the hook
    assert rec.z is None


def test_without_a_gpu_the_call_raises_and_never_computes():
    from george_b200 import _lib
    try:
        lib = _lib.load()
    except ImportError:
        pytest.skip("the library is not built")
    if lib.bgp_device_count() > 0:
        pytest.skip("a GPU is present")
    from george_b200.solvers._hodlr import HODLRSolver
    s = HODLRSolver()
    with pytest.raises(RuntimeError, match="not been computed"):
        s.apply_symmetric_factor(np.zeros(5))
    with pytest.raises(RuntimeError, match="not been computed"):
        s.symmetric_log_determinant
    from george_b200 import kernels
    with pytest.raises(_lib.BGPError):
        s.compute(kernels.Matern32Kernel(1.0), np.linspace(0, 1, 5)[:, None], np.ones(5), min_size=2)
    # the handle was never computed: the symmetric factor refuses rather than computing anything
    status = lib.bgp_hodlr_sym_factor(s._ptr)
    assert status == _lib.BGP_ERR_NOT_COMPUTED
