# -*- coding: utf-8 -*-
"""``GP.fisher_information`` on the host (no GPU), around stub dense solvers with a fixed SPD ``K^-1`` and a fixed kernel
gradient tensor: the output layout and shape, frozen parameters, the mean block with a non-constant mean and the
white-noise block with a non-constant white-noise model, ``quiet``, the GP's state after a call, the host route (a
plug-in without ``fisher_terms`` and a hook returning ``None``) against a numpy evaluation of the formula, and ``(grad,
F)``'s ``grad`` against ``grad_log_likelihood``.  The device arithmetic is tested in tests/test_gpu_fisher.py."""
import numpy as np
import pytest
from numpy.linalg import LinAlgError

N = 9
_rng = np.random.default_rng(11)
_G = _rng.standard_normal((N, N))
KINV = _G.dot(_G.T) / N + np.eye(N)                 # SPD, exactly symmetric
P_ALL = 4                                            # 1.3 * ExpSquared + 0.4 * Exp: two parameters each
DK = _rng.standard_normal((N, N, P_ALL))
DK = DK + DK.transpose(1, 0, 2)                      # each plane exactly symmetric

MEAN_NAN = 50.0  # LineMean slope above it: the mean gradient is NaN


def _line_mean(m, b):
    from george_b200.modeling import Model

    class LineMean(Model):
        parameter_names = ("m", "b")

        def get_value(self, x):
            return self.m * np.asarray(x).flatten() + self.b

        def compute_gradient(self, x):
            x = np.asarray(x).flatten()
            g = np.vstack([x, np.ones_like(x)])
            return g if self.m <= MEAN_NAN else g * np.nan

    return LineMean(m=m, b=b)


def _log_linear_noise(a, s):
    from george_b200.modeling import Model

    class LogLinearNoise(Model):
        parameter_names = ("a", "s")

        def get_value(self, x):
            return self.a + self.s * np.asarray(x).flatten()

        def compute_gradient(self, x):
            x = np.asarray(x).flatten()
            return np.vstack([np.ones_like(x), x])

    return LogLinearNoise(a=a, s=s)


def _contract(B, which):
    return np.einsum("ij,ijq->q", B, DK) * (np.asarray(which) != 0)


class _Stub(object):
    """A dense solver plug-in with ``K^-1 = KINV`` and the kernel gradient ``DK``; its ``fisher_terms`` hook evaluates
    the rows on the host.  ``fail`` makes the hooks raise ValueError; every hook call is recorded in ``calls``."""
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
        self.log_determinant = 1.0
        self.computed = True

    def apply_inverse(self, y, in_place=False):
        return KINV.dot(np.asarray(y, dtype=np.float64))

    def dot_solve(self, y):
        return float(np.dot(y, KINV.dot(y)))

    def get_inverse(self):
        return KINV.copy()

    def _terms(self, r, which):
        if _Stub.fail:
            raise ValueError("stub failure")
        alpha = KINV.dot(r)
        A = np.outer(alpha, alpha) - KINV
        return alpha, _contract(A, which), np.diag(A).copy()

    def grad_terms(self, r, which):
        _Stub.calls.append(("grad_terms", list(which)))
        return self._terms(r, which)

    def fisher_terms(self, r, which, v, prod_ms=None):
        _Stub.calls.append(("fisher_terms", r is not None, list(which), len(v)))
        terms = None if r is None else self._terms(r, which)
        if _Stub.fail:
            raise ValueError("stub failure")
        planes = [KINV.dot(DK[:, :, p]).dot(KINV) for p in range(len(which)) if which[p]]
        planes += [KINV.dot(vk[:, None] * KINV) for vk in v]
        rows = np.array([_contract(B, which) for B in planes]).reshape(len(planes), len(which))
        rdiag = np.array([np.diag(B) for B in planes]).reshape(len(planes), N)
        return terms, rows, rdiag


class _Plugin(_Stub):
    """A plug-in without the hook: the GP takes its host route."""
    fisher_terms = None


class _Pickled(_Stub):
    """A hook that returns ``None``, as a dense solver restored from a pickle does."""

    def fisher_terms(self, r, which, v, prod_ms=None):
        _Stub.calls.append(("fisher_terms", r is not None, list(which), len(v)))
        return None


@pytest.fixture(autouse=True)
def _reset(monkeypatch):
    _Stub.calls, _Stub.fail, _Stub.fail_compute = [], False, False
    from george_b200 import kernels
    from george_b200.kernel_interface import KernelInterface
    # the host route's kernel gradients, without a device
    monkeypatch.setattr(kernels.Kernel, "get_gradient",
                        lambda self, x1, x2=None, include_frozen=False: DK[:, :, self.unfrozen_mask])
    monkeypatch.setattr(KernelInterface, "gradient_contract", lambda self, which, x, A: _contract(A, which))
    yield


def _gp(solver=_Stub, **kwargs):
    import george_b200 as george
    from george_b200 import kernels
    k = 1.3 * kernels.ExpSquaredKernel(0.7) + 0.4 * kernels.ExpKernel(1.5)
    gp = george.GP(k, solver=solver, **kwargs)
    rng = np.random.default_rng(5)
    x = np.sort(rng.uniform(0, 3, N))
    gp.compute(x, 0.1 + 0.05 * rng.random(N))
    return gp, x, rng.standard_normal(N)


def _reference(gp, x):
    """F from the formula, one entry at a time: dmu_p K^-1 dmu_q for the mean, 1/2 tr(K^-1 dK_a K^-1 dK_b) for the rest."""
    n_mean, n_wn = len(gp.mean), len(gp.white_noise)
    dmu = gp.mean.get_gradient(x).reshape(n_mean, N) if n_mean else np.zeros((0, N))
    dks = []
    if n_wn:
        wn = gp.white_noise.get_value(x).flatten()
        dwn = gp.white_noise.get_gradient(x).reshape(n_wn, N)
        dks += [np.diag(np.exp(wn) * dwn[k]) for k in range(n_wn)]
    dks += [DK[:, :, p] for p in np.flatnonzero(gp.kernel.unfrozen_mask)]
    size = len(gp)
    F = np.zeros((size, size))
    F[:n_mean, :n_mean] = dmu.dot(KINV).dot(dmu.T)
    for a, da in enumerate(dks):
        for b, db in enumerate(dks):
            F[n_mean + a, n_mean + b] = 0.5 * np.trace(KINV.dot(da).dot(KINV).dot(db))
    return F


MODELS = [
    dict(),
    dict(mean=0.4, fit_mean=True),
    dict(white_noise=-3.0, fit_white_noise=True),
    dict(mean=0.4, fit_mean=True, white_noise=-3.0, fit_white_noise=True, fit_kernel=False),
    dict(mean="line", fit_mean=True, white_noise="loglinear", fit_white_noise=True),
]


def _models(kwargs):
    kwargs = dict(kwargs)
    if kwargs.get("mean") == "line":
        kwargs["mean"] = _line_mean(0.3, -0.2)
    if kwargs.get("white_noise") == "loglinear":
        kwargs["white_noise"] = _log_linear_noise(-2.5, 0.4)
    return kwargs


@pytest.mark.parametrize("solver", [_Stub, _Plugin, _Pickled])
@pytest.mark.parametrize("kwargs", MODELS)
def test_formula_layout_and_shape(solver, kwargs):
    gp, x, y = _gp(solver, **_models(kwargs))
    F = gp.fisher_information()
    assert F.shape == (len(gp), len(gp)) and F.dtype == np.float64
    assert np.array_equal(F, F.T)
    ref = _reference(gp, x)
    assert np.allclose(F, ref, rtol=1e-12, atol=1e-12 * np.abs(ref).max())
    assert np.array_equal(F, gp.fisher_information())


def test_device_route_without_y_skips_alpha():
    gp, x, y = _gp(white_noise=-3.0, fit_white_noise=True)
    gp.fisher_information()
    assert _Stub.calls == [("fisher_terms", False, [1] * P_ALL, 1)]
    gp.fisher_information(y)
    assert _Stub.calls[-1] == ("fisher_terms", True, [1] * P_ALL, 1)


def test_mean_only_needs_no_hook():
    gp, x, y = _gp(mean=_line_mean(0.3, -0.2), fit_mean=True, fit_kernel=False)
    F = gp.fisher_information()
    assert F.shape == (2, 2) and _Stub.calls == []
    dmu = np.vstack([x, np.ones_like(x)])
    assert np.allclose(F, dmu.dot(KINV).dot(dmu.T), rtol=1e-13)


@pytest.mark.parametrize("solver", [_Stub, _Plugin, _Pickled])
@pytest.mark.parametrize("kwargs", MODELS)
def test_grad_is_grad_log_likelihood(solver, kwargs):
    gp, x, y = _gp(solver, **_models(kwargs))
    grad, F = gp.fisher_information(y)
    assert np.array_equal(grad, gp.grad_log_likelihood(y))
    assert np.array_equal(F, gp.fisher_information())


@pytest.mark.parametrize("solver", [_Stub, _Plugin])
def test_frozen_parameters(solver):
    gp, x, y = _gp(solver, mean=0.4, fit_mean=True, white_noise=-3.0, fit_white_noise=True)
    full = gp.fisher_information()
    gp.freeze_parameter("kernel:k1:k2:metric:log_M_0_0")
    mask = gp.kernel.unfrozen_mask
    assert mask.sum() == P_ALL - 1
    grad, F = gp.fisher_information(y)
    assert F.shape == (len(gp), len(gp)) == (2 + P_ALL - 1, 2 + P_ALL - 1)
    keep = np.concatenate([[True, True], mask])
    assert np.allclose(F, full[np.ix_(keep, keep)], rtol=1e-13, atol=1e-14 * np.abs(full).max())
    if solver is _Stub:
        assert _Stub.calls[-1] == ("fisher_terms", True, [int(m) for m in mask], 1)
    assert np.array_equal(grad, gp.grad_log_likelihood(y))


def test_cross_blocks_are_zero():
    gp, x, y = _gp(mean=_line_mean(0.3, -0.2), fit_mean=True)
    F = gp.fisher_information()
    assert not F[:2, 2:].any() and not F[2:, :2].any()


def test_quiet_absorbs_a_hook_failure():
    gp, x, y = _gp(mean=0.4, fit_mean=True)
    _Stub.fail = True
    with pytest.raises(ValueError, match="stub failure"):
        gp.fisher_information()
    F = gp.fisher_information(quiet=True)
    assert F.shape == (len(gp), len(gp)) and not F.any()
    grad, F = gp.fisher_information(y, quiet=True)
    assert grad.shape == (len(gp),) and not grad.any() and not F.any()


def test_quiet_absorbs_a_model_failure():
    gp, x, y = _gp(mean=_line_mean(MEAN_NAN + 1.0, 0.0), fit_mean=True)
    with pytest.raises(ValueError, match="mean gradient"):
        gp.fisher_information()
    assert not gp.fisher_information(quiet=True).any()
    grad, F = gp.fisher_information(y, quiet=True)
    assert not grad.any() and not F.any()


def test_quiet_absorbs_a_failed_factorisation():
    gp, x, y = _gp()
    gp.set_parameter_vector(gp.get_parameter_vector() + 0.1)  # dirty: the next call refactorises
    _Stub.fail_compute = True
    with pytest.raises(LinAlgError):
        gp.fisher_information()
    F = gp.fisher_information(quiet=True)
    assert F.shape == (P_ALL, P_ALL) and not F.any()
    grad, F = gp.fisher_information(y, quiet=True)
    assert not grad.any() and not F.any()
    assert _Stub.calls == []


def test_requires_compute():
    import george_b200 as george
    from george_b200 import kernels
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0), solver=_Stub)
    with pytest.raises(RuntimeError, match="compute"):
        gp.fisher_information()


def test_state_is_unchanged():
    gp, x, y = _gp(mean=_line_mean(0.3, -0.2), fit_mean=True, white_noise=_log_linear_noise(-2.5, 0.4),
                   fit_white_noise=True)
    gp.log_likelihood(y)
    solver, vec = gp.solver, gp.get_parameter_vector().copy()
    alpha, cached_y = gp._alpha, gp._y
    gp.fisher_information(y)
    gp.fisher_information()
    assert gp.solver is solver and gp.computed
    assert np.array_equal(gp.get_parameter_vector(), vec)
    assert gp._alpha is alpha and gp._y is cached_y
