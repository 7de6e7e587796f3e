# -*- coding: utf-8 -*-
"""GP.batch_log_likelihood and GP.batch_grad_log_likelihood on the host (no GPU), around a stub solver whose
``batch_log_likelihood``, ``batch_grad_terms``, ``dot_solve`` and ``grad_terms`` return fixed arrays, a function of the
member's kernel parameters, noise and residual:

* batch == loop bit for bit, with ``quiet`` on and off and (gradient) ``return_log_likelihood`` on and off, for every
  failure kind a member can meet: a white-noise model that raises, a factorisation that fails, an invalid program, a
  non-finite mean, a mean model that raises, a non-finite residual and a NaN mean gradient;
* the exception the loop meets first is the one raised;
* the gradient layout with frozen parameters, the GP's state after the call, and the order of the calls into the mean
  and white-noise models.

``y`` is float64 throughout: with it the batch's one residual for value and gradient is the loop's for both.
"""
import math

import numpy as np
import pytest
from numpy.linalg import LinAlgError

N = 12

ALPHA = np.linspace(-1.0, 1.0, N)
DIAG_A = np.linspace(-0.2, 0.3, N)
FAIL_LOG_CONSTANT = 5.0      # kernel parameter 0 above it: the factorisation fails with info 3
INVALID_LOG_CONSTANT = -7.0  # kernel parameter 0 equal to it: the member's program is invalid (info -1)
NOISE_LIMIT = 10.0           # white noise "a" above it: ValueError; below minus it: RuntimeError
MEAN_LIMIT = 10.0            # mean "b" above it: ValueError; below minus it: RuntimeError
SLOPE_LIMIT = 100.0          # mean "m" above it: the mean gradient is NaN

CALLS = []  # (model, method, parameters) of every call into the mean and white-noise models, in order


def _line_mean(m, b):
    from george_b200.modeling import Model

    class LineMean(Model):
        parameter_names = ("m", "b")

        def get_value(self, x):
            CALLS.append(("mean", "value", (self.m, self.b)))
            if self.b > MEAN_LIMIT:
                raise ValueError("mean intercept out of range")
            if self.b < -MEAN_LIMIT:
                raise RuntimeError("mean model broke")
            return self.m * np.asarray(x).flatten() + self.b

        def compute_gradient(self, x):
            CALLS.append(("mean", "gradient", (self.m, self.b)))
            x = np.asarray(x).flatten()
            g = np.vstack([x, np.ones_like(x)])
            return g if self.m <= SLOPE_LIMIT else g * np.nan

    return LineMean(m=m, b=b)


def _log_linear_noise(a, s):
    from george_b200.modeling import Model

    class LogLinearNoise(Model):
        parameter_names = ("a", "s")

        def get_value(self, x):
            CALLS.append(("noise", "value", (self.a, self.s)))
            if self.a > NOISE_LIMIT:
                raise ValueError("white noise out of range")
            if self.a < -NOISE_LIMIT:
                raise RuntimeError("white noise model broke")
            return self.a + self.s * np.asarray(x).flatten()

        def compute_gradient(self, x):
            CALLS.append(("noise", "gradient", (self.a, self.s)))
            x = np.asarray(x).flatten()
            return np.vstack([np.ones_like(x), x])

    return LogLinearNoise(a=a, s=s)


# The stub's terms of one member: kernel parameters kp, noise yerr, residual r.  Sums go through math.fsum, which
# rounds once whatever the memory layout, so a batch row and a single call give the same bits.
def _log_det(kp, yerr):
    return kp[0] + 2.0 * kp[1] + 0.01 * math.fsum(yerr)


def _quad(kp, r):
    return math.fsum(r * r) / (1.0 + kp[1] ** 2)


def _grad_terms(kp, yerr, r, which):
    g = (10.0 * np.arange(len(which)) + 1.0) * kp[0] * (np.asarray(which) != 0)
    return ALPHA * kp[0] + r / yerr, g, DIAG_A * kp[1] * yerr


def _info(kp):
    return 3 if kp[0] > FAIL_LOG_CONSTANT else (-1 if kp[0] == INVALID_LOG_CONSTANT else 0)


class _StubSolver(object):
    """The single and batched hooks from the functions above; compute fails as the batch's info says."""

    batch_calls = []

    def __init__(self, kernel, **kwargs):
        self.kernel = kernel
        self.computed = False

    def compute(self, x, yerr):
        self._kp = self.kernel.get_parameter_vector(include_frozen=True)
        info = _info(self._kp)
        if info > 0:
            raise LinAlgError("%d-th leading minor of the array is not positive definite" % info)
        if info < 0:
            raise ValueError("invalid kernel")
        self._yerr = np.array(yerr)
        self.log_determinant = _log_det(self._kp, self._yerr)
        self.computed = True

    def apply_inverse(self, y, in_place=False):
        raise AssertionError("the hook route must not form K^-1")

    def dot_solve(self, r):
        from george_b200.solvers.basic import _check_finite
        _check_finite(r)
        return _quad(self._kp, np.asarray(r))

    def grad_terms(self, r, which):
        from george_b200.solvers.basic import _check_finite
        _check_finite(r)
        return _grad_terms(self._kp, self._yerr, np.asarray(r), which)

    @staticmethod
    def batch_log_likelihood(spec, params, x, yerr, r):
        _StubSolver.batch_calls.append(("ll", np.array(params), np.array(r), None))
        info = np.array([_info(p) for p in params], dtype=np.int32)
        log_det = np.array([_log_det(p, e) for p, e in zip(params, yerr)])
        quad = np.array([_quad(p, rb) for p, rb in zip(params, r)])
        log_det[info != 0] = quad[info != 0] = np.nan
        return log_det, quad, info

    @staticmethod
    def batch_grad_terms(spec, params, x, yerr, r, which):
        log_det, quad, info = _StubSolver.batch_log_likelihood(spec, params, x, yerr, r)
        _StubSolver.batch_calls[-1] = ("grad", np.array(params), np.array(r), np.array(which))
        rows = [_grad_terms(p, e, rb, which) for p, e, rb in zip(params, yerr, r)]
        alpha, g, diag = [np.stack([row[k] for row in rows]) for k in range(3)]
        for a in (alpha, g, diag):
            a[info != 0] = np.nan
        return log_det, quad, alpha, g, diag, info


def _data(n=N, seed=3):
    rng = np.random.default_rng(seed)
    x = np.sort(rng.uniform(0, 5, n))
    yerr = 0.2 + 0.1 * rng.random(n)
    y = 0.4 * x - 0.3 + 0.5 * rng.standard_normal(n)
    return x, yerr, y


def _stub_gp(constant=False, freeze=()):
    """Vector: (m, b, a, s, log_constant, log_M), or with ``constant`` (mean, log white noise, log_constant, log_M)."""
    import george_b200 as george
    from george_b200 import kernels
    kernel = 2.0 * kernels.ExpSquaredKernel(1.5)
    if constant:
        gp = george.GP(kernel, mean=0.2, fit_mean=True, white_noise=np.log(0.05), fit_white_noise=True,
                       solver=_StubSolver)
    else:
        gp = george.GP(kernel, mean=_line_mean(0.3, -0.1), fit_mean=True, white_noise=_log_linear_noise(-2.0, 0.1),
                       fit_white_noise=True, solver=_StubSolver)
    for name in freeze:
        gp.freeze_parameter(name)
    x, yerr, y = _data()
    gp.compute(x, yerr)
    _StubSolver.batch_calls = []
    return gp, y


def _vectors(gp, nb=5, seed=4):
    rng = np.random.default_rng(seed)
    return gp.get_parameter_vector() + 0.1 * rng.standard_normal((nb, len(gp)))


METHODS = ["ll", "grad", "grad_ll"]


def _loop(gp, vecs, y, method, quiet):
    """The per-vector path the batch stands for: the values, the gradients, or (values, gradients)."""
    p0 = gp.get_parameter_vector()
    ll, grad = [], []
    try:
        for v in vecs:
            gp.set_parameter_vector(v)
            if method != "grad":
                ll.append(gp.log_likelihood(y, quiet=quiet))
            if method != "ll":
                grad.append(gp.grad_log_likelihood(y, quiet=quiet))
    finally:
        gp.set_parameter_vector(p0)
    ll = np.array(ll, dtype=np.float64)
    grad = np.stack(grad) if grad else None
    return ll if method == "ll" else (grad if method == "grad" else (ll, grad))


def _batch(gp, vecs, y, method, quiet):
    if method == "ll":
        return gp.batch_log_likelihood(vecs, y, quiet=quiet)
    return gp.batch_grad_log_likelihood(vecs, y, quiet=quiet, return_log_likelihood=method == "grad_ll")


def _same(got, want):
    if isinstance(want, tuple):
        return all(_same(a, b) for a, b in zip(got, want))
    return got.shape == want.shape and got.dtype == want.dtype and np.array_equal(got, want, equal_nan=True)


def _state(gp):
    return (gp.get_parameter_vector(include_frozen=True).copy(), gp.computed, gp.solver, gp._alpha, gp._y, gp._const,
            [m.dirty for m in gp.models.values()])


def _assert_state(gp, st):
    now = _state(gp)
    assert np.array_equal(st[0], now[0])
    assert now[1] == st[1] and now[5] == st[5] and now[6] == st[6]
    assert now[2] is st[2] and now[3] is st[3] and now[4] is st[4]


def _outcome(gp, vecs, y, method, quiet):
    """``("ok", result)`` or ``("raise", exception)`` of the batch, the GP checked to be left as it was, and the same of
    the loop."""
    gp.recompute(quiet=True)
    st = _state(gp)
    _StubSolver.batch_calls = []
    try:
        got = ("ok", _batch(gp, vecs, y, method, quiet))
    except Exception as exc:
        got = ("raise", exc)
    _assert_state(gp, st)
    assert [c[0] for c in _StubSolver.batch_calls] == ["ll" if method == "ll" else "grad"]  # the batched path ran
    try:
        want = ("ok", _loop(gp, vecs, y, method, quiet))
    except Exception as exc:
        want = ("raise", exc)
    gp.recompute(quiet=True)
    return got, want


def _assert_same_outcome(got, want):
    assert got[0] == want[0], (got, want)
    if got[0] == "raise":
        assert type(got[1]) is type(want[1]) and str(got[1]) == str(want[1])
    else:
        assert _same(got[1], want[1])


# ---- no failures ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("constant", [False, True])
@pytest.mark.parametrize("quiet", [False, True])
@pytest.mark.parametrize("method", METHODS)
def test_stub_matches_the_loop(method, quiet, constant):
    gp, y = _stub_gp(constant=constant)
    got, want = _outcome(gp, _vectors(gp), y, method, quiet)
    assert got[0] == "ok"
    _assert_same_outcome(got, want)
    out = got[1] if method == "grad_ll" else (got[1], None)
    if method != "grad":
        assert np.all(np.isfinite(out[0]))
    if method != "ll":
        grad = out[1] if method == "grad_ll" else got[1]
        assert grad.shape == (5, len(gp)) and np.all(grad != 0.0)


def test_stub_gradient_layout():
    """Mean ``dmu . alpha``, white noise ``1/2 sum exp(wn) diagA dwn``, kernel ``1/2 g``; ll from log_det and quad."""
    gp, y = _stub_gp()
    x, yerr2 = gp._x[:, 0], gp._yerr2
    vecs = _vectors(gp, nb=3)
    ll, grad = gp.batch_grad_log_likelihood(vecs, y, return_log_likelihood=True)
    assert np.array_equal(_StubSolver.batch_calls[-1][3], [1, 1])
    for b, v in enumerate(vecs):
        m, c, a, s, lc, lm = v
        wn = a + s * x
        sigma = np.sqrt(yerr2 + np.exp(wn))
        r = y - (m * x + c)
        alpha = ALPHA * lc + r / sigma
        ref = np.concatenate([
            [np.dot(x, alpha), np.sum(alpha)],
            0.5 * np.array([np.sum(np.exp(wn) * DIAG_A * lm * sigma), np.sum(np.exp(wn) * DIAG_A * lm * sigma * x)]),
            0.5 * np.array([lc, 11.0 * lc]),
        ])
        assert np.allclose(grad[b], ref, rtol=1e-13, atol=1e-13), b
        want = -0.5 * (N * np.log(2 * np.pi) + lc + 2.0 * lm + 0.01 * np.sum(sigma)) \
            - 0.5 * np.sum(r * r) / (1.0 + lm ** 2)
        assert np.isclose(ll[b], want, rtol=1e-13), b


@pytest.mark.parametrize("method", ["grad", "grad_ll"])
def test_stub_frozen_parameters(method):
    gp, y = _stub_gp(freeze=("kernel:k1:log_constant", "mean:b", "white_noise:s"))
    assert len(gp) == 3
    vecs = _vectors(gp, nb=4)
    got, want = _outcome(gp, vecs, y, method, False)
    _assert_same_outcome(got, want)
    grad = got[1] if method == "grad" else got[1][1]
    assert grad.shape == (4, 3)
    _, full, _, which = _StubSolver.batch_calls[0]
    assert np.array_equal(which, [0, 1])  # which covers every kernel parameter
    assert np.all(full[:, 0] == np.log(2.0)) and np.array_equal(full[:, 1], vecs[:, 2])


# ---- failures ------------------------------------------------------------------------------------------------------

# failure kind: (constant-mean GP, full-vector entry, value); entry None: y[2] becomes inf for every member
FAILURES = {
    "white_noise": (False, 2, NOISE_LIMIT + 1.0),
    "white_noise_runtime_error": (False, 2, -NOISE_LIMIT - 1.0),
    "factorisation": (False, 4, FAIL_LOG_CONSTANT + 1.0),
    "invalid_program": (False, 4, INVALID_LOG_CONSTANT),
    "nan_constant_mean": (True, 0, np.nan),
    "nan_mean": (False, 0, np.nan),
    "mean_raises": (False, 1, MEAN_LIMIT + 1.0),
    "mean_runtime_error": (False, 1, -MEAN_LIMIT - 1.0),
    "nonfinite_residual": (False, None, None),
    "nan_mean_gradient": (False, 0, SLOPE_LIMIT + 1.0),
}
# with quiet, what the failing members get: "swallowed" (-inf, zero gradient), "raise" or "fine" (the method does not
# look at what fails); without quiet a failure that is not "fine" raises
QUIET = {
    "white_noise": dict(ll="swallowed", grad="swallowed", grad_ll="swallowed"),
    "white_noise_runtime_error": dict(ll="raise", grad="raise", grad_ll="raise"),
    "factorisation": dict(ll="swallowed", grad="swallowed", grad_ll="swallowed"),
    "invalid_program": dict(ll="swallowed", grad="swallowed", grad_ll="swallowed"),
    "nan_constant_mean": dict(ll="swallowed", grad="swallowed", grad_ll="swallowed"),
    "nan_mean": dict(ll="swallowed", grad="swallowed", grad_ll="swallowed"),
    "mean_raises": dict(ll="raise", grad="swallowed", grad_ll="raise"),          # a ValueError not about the mean
    "mean_runtime_error": dict(ll="raise", grad="raise", grad_ll="raise"),
    "nonfinite_residual": dict(ll="raise", grad="swallowed", grad_ll="raise"),    # the solver's ValueError
    "nan_mean_gradient": dict(ll="fine", grad="swallowed", grad_ll="swallowed"),  # (grad_ll: a finite ll, zero grad)
}


def _failing(failure, members=(1, 3)):
    constant, entry, value = FAILURES[failure]
    gp, y = _stub_gp(constant=constant)
    vecs = _vectors(gp, nb=5, seed=6)
    if entry is None:
        y = y.copy()
        y[2] = np.inf
    else:
        vecs[list(members), entry] = value
    return gp, vecs, y


@pytest.mark.parametrize("quiet", [False, True])
@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("failure", sorted(FAILURES))
def test_failures_match_the_loop(failure, method, quiet):
    gp, vecs, y = _failing(failure)
    got, want = _outcome(gp, vecs, y, method, quiet)
    _assert_same_outcome(got, want)
    expect = QUIET[failure][method]
    if expect != "fine" and not quiet:
        expect = "raise"
    assert got[0] == ("raise" if expect == "raise" else "ok"), (failure, method, quiet, got)
    if got[0] == "raise":
        return
    failed = list(range(5)) if FAILURES[failure][1] is None else [1, 3]
    others = [b for b in range(5) if b not in failed]
    ll = got[1] if method == "ll" else (got[1][0] if method == "grad_ll" else None)
    grad = None if method == "ll" else (got[1] if method == "grad" else got[1][1])
    if ll is not None:
        assert np.all(np.isfinite(ll[others]))
        assert np.all(np.isneginf(ll[failed]) == (expect == "swallowed" and failure != "nan_mean_gradient"))
    if grad is not None:
        assert np.all(grad[others] != 0.0)
        assert np.all((grad[failed] == 0.0) == (expect == "swallowed"))


@pytest.mark.parametrize("method", METHODS)
def test_the_first_failing_member_decides(method):
    """Two failure kinds in two members: the one the loop meets first is raised, whatever its kind."""
    for first, second in (("nan_mean", "factorisation"), ("factorisation", "nan_mean"),
                          ("white_noise", "mean_raises"), ("mean_raises", "white_noise")):
        gp, y = _stub_gp()
        vecs = _vectors(gp, nb=5, seed=6)
        for b, failure in ((1, first), (3, second)):
            _, entry, value = FAILURES[failure]
            vecs[b, entry] = value
        for quiet in (False, True):
            got, want = _outcome(gp, vecs, y, method, quiet)
            _assert_same_outcome(got, want)
            if not quiet:
                assert got[0] == "raise"
                assert type(got[1]) is {"nan_mean": ValueError, "factorisation": LinAlgError,
                                        "white_noise": ValueError, "mean_raises": ValueError}[first]


# ---- the calls into the mean and white-noise models ----------------------------------------------------------------

def test_model_call_order():
    """The batch evaluates the white noise of every member, then every member's mean, then member by member the mean
    gradient and the white noise with its gradient; a failing member skips its gradient calls."""
    gp, y = _stub_gp()
    vecs = _vectors(gp, nb=4)
    vecs[2, 4] = FAIL_LOG_CONSTANT + 1.0
    gp.recompute()
    del CALLS[:]
    gp.batch_grad_log_likelihood(vecs, y, quiet=True)
    mean = [("mean", tuple(v[:2])) for v in vecs]
    noise = [("noise", tuple(v[2:4])) for v in vecs]
    want = [(n[0], "value", n[1]) for n in noise] + [(m[0], "value", m[1]) for m in mean]
    for b in (0, 1, 3):
        want += [(mean[b][0], "gradient", mean[b][1]), (noise[b][0], "value", noise[b][1]),
                 (noise[b][0], "gradient", noise[b][1])]
    assert CALLS == want
    del CALLS[:]
