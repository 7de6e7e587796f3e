# -*- coding: utf-8 -*-
"""GP.batch_loo_predict, GP.batch_loo_log_likelihood and GP.batch_grad_loo_log_likelihood on the host (no GPU).

* the argument checks that run before any device call, the empty results, the error raised without a device;
* the GP layer around a stub solver whose ``batch_loo_terms`` and ``loo_terms`` return fixed arrays, a function of the
  member's kernel parameters and residual: the gradient layout with frozen parameters, a fitted mean and a non-constant
  white-noise model, ``quiet`` member by member for every failure kind, the first loop error, the GP's state;
* the per-vector loop taken by ``TrivialSolver``, a ``HODLRSolver``-typed GP and, for the gradient, more than 64 kernel
  parameters.
"""
import numpy as np
import pytest
from numpy.linalg import LinAlgError

N = 12

ALPHA = np.linspace(-1.0, 1.0, N)
D = np.linspace(1.0, 2.0, N)
BETA = np.linspace(0.5, -0.5, N)
DIAG_A = np.linspace(-0.2, 0.3, N)
FAIL_LOG_CONSTANT = 5.0      # kernel parameter 0 above it: the factorisation fails with info 3
INVALID_LOG_CONSTANT = -7.0  # kernel parameter 0 equal to it: the member's program is invalid (info -1)
NOISE_LIMIT = 10.0           # white noise "a" above it: the white-noise model raises
SLOPE_LIMIT = 100.0          # mean "m" above it: the mean gradient is NaN


def _line_mean(m, b):
    from george_b200.modeling import Model

    class LineMean(Model):
        parameter_names = ("m", "b")

        def get_value(self, x):
            return self.m * np.asarray(x).flatten() + self.b

        def compute_gradient(self, x):
            x = np.asarray(x).flatten()
            g = np.vstack([x, np.ones_like(x)])
            return g if self.m <= SLOPE_LIMIT else g * np.nan

    return LineMean(m=m, b=b)


def _log_linear_noise(a, s):
    from george_b200.modeling import Model

    class LogLinearNoise(Model):
        parameter_names = ("a", "s")

        def get_value(self, x):
            if self.a > NOISE_LIMIT:
                raise ValueError("white noise out of range")
            return self.a + self.s * np.asarray(x).flatten()

        def compute_gradient(self, x):
            x = np.asarray(x).flatten()
            return np.vstack([np.ones_like(x), x])

    return LogLinearNoise(a=a, s=s)


def _terms(kp, r, which):
    """The stub's LOO terms of one member: kernel parameters ``kp``, residual ``r``."""
    alpha = ALPHA * kp[0] + r
    d = D + kp[1]
    if which is None:
        return alpha, d
    g = (10.0 * np.arange(len(which)) + 1.0) * kp[0] * (np.asarray(which) != 0)
    return alpha, d, BETA * kp[0], g, DIAG_A * kp[1]


def _info(kp):
    return 3 if kp[0] > FAIL_LOG_CONSTANT else (-1 if kp[0] == INVALID_LOG_CONSTANT else 0)


class _StubSolver(object):
    """loo_terms and batch_loo_terms from _terms; compute fails as the batch's info says."""

    batch_calls = []

    def __init__(self, kernel, **kwargs):
        self.kernel = kernel
        self.computed = False

    def compute(self, x, yerr):
        info = _info(self.kernel.get_parameter_vector(include_frozen=True))
        if info > 0:
            raise LinAlgError("%d-th leading minor of the array is not positive definite" % info)
        if info < 0:
            raise ValueError("invalid kernel")
        self.log_determinant = 0.0
        self.computed = True

    def apply_inverse(self, y, in_place=False):
        raise AssertionError("the hook route must not form K^-1")

    def dot_solve(self, y):
        return 0.0

    def loo_terms(self, r, which=None):
        """BasicSolver.loo_terms' checks: a non-finite residual, then (gradient) a d that is not finite and positive."""
        from george_b200.solvers.basic import NONFINITE_RHS
        if not np.all(np.isfinite(r)):
            raise ValueError(NONFINITE_RHS)
        terms = _terms(self.kernel.get_parameter_vector(include_frozen=True), np.asarray(r), which)
        bad = np.flatnonzero(~(np.isfinite(terms[1]) & (terms[1] > 0)))
        if which is not None and bad.size:
            raise ValueError("leave-one-out: diag(K^-1) at point %d is %g, not a finite positive number"
                             % (bad[0], terms[1][bad[0]]))
        return terms

    @staticmethod
    def batch_loo_terms(spec, params, x, yerr, r, which=None):
        _StubSolver.batch_calls.append((np.array(params), np.array(r), None if which is None else np.array(which)))
        rows = [_terms(p, rb, which) for p, rb in zip(params, r)]
        out = [np.stack([row[k] for row in rows]) for k in range(len(rows[0]))]
        info = np.array([_info(p) for p in params], dtype=np.int32)
        for a in out:
            a[info != 0] = np.nan
        return tuple(out) + (info,)


def _data(n=N, seed=3):
    rng = np.random.default_rng(seed)
    x = np.sort(rng.uniform(0, 5, n))
    yerr = 0.2 + 0.1 * rng.random(n)
    y = 0.4 * x - 0.3 + 0.5 * rng.standard_normal(n)
    return x, yerr, y


def _stub_gp(freeze=(), solver=_StubSolver):
    import george_b200 as george
    from george_b200 import kernels
    kernel = 2.0 * kernels.ExpSquaredKernel(1.5)  # parameters: k1:log_constant, k2:metric:log_M_0_0
    gp = george.GP(kernel, mean=_line_mean(0.3, -0.1), fit_mean=True, white_noise=_log_linear_noise(-2.0, 0.1),
                   fit_white_noise=True, solver=solver)
    for name in freeze:
        gp.freeze_parameter(name)
    x, yerr, y = _data()
    gp.compute(x, yerr)
    _StubSolver.batch_calls = []
    return gp, y


def _vectors(gp, nb=5, seed=4):
    rng = np.random.default_rng(seed)
    return gp.get_parameter_vector() + 0.1 * rng.standard_normal((nb, len(gp)))


def _loop(gp, vecs, y, kind, quiet=False):
    """The per-vector path the batch stands for: (mu, var), the values, or (values, gradients)."""
    p0 = gp.get_parameter_vector()
    res = []
    try:
        for v in vecs:
            gp.set_parameter_vector(v)
            if kind == "predict":
                res.append(gp.loo_predict(y))
            elif kind == "value":
                res.append(gp.loo_log_likelihood(y, quiet=quiet))
            else:
                res.append(gp.grad_loo_log_likelihood(y, quiet=quiet, return_value=True))
    finally:
        gp.set_parameter_vector(p0)
    if kind == "value":
        return np.array(res)
    return np.stack([r[0] for r in res]), np.stack([r[1] for r in res])


def _batch(gp, vecs, y, kind, quiet=False):
    if kind == "predict":
        return gp.batch_loo_predict(vecs, y)
    if kind == "value":
        return gp.batch_loo_log_likelihood(vecs, y, quiet=quiet)
    value, grad = gp.batch_grad_loo_log_likelihood(vecs, y, quiet=quiet, return_value=True)
    assert np.array_equal(grad, gp.batch_grad_loo_log_likelihood(vecs, y, quiet=quiet))
    return value, grad


def _same(got, want):
    if isinstance(want, tuple):
        return all(_same(a, b) for a, b in zip(got, want))
    return got.shape == want.shape and np.array_equal(got, want, equal_nan=True)


def _state(gp):
    return (gp.get_parameter_vector(include_frozen=True).copy(), gp.computed, gp.solver, gp._alpha, gp._y, gp._const,
            [m.dirty for m in gp.models.values()])


def _assert_state(gp, st):
    now = _state(gp)
    assert np.array_equal(st[0], now[0])
    assert now[1] == st[1] and now[5] == st[5] and now[6] == st[6]
    assert now[2] is st[2] and now[3] is st[3] and now[4] is st[4]


def _check(gp, vecs, y, kind, quiet=False):
    """batch == loop bit for bit, the GP left as it was; returns the batch's result."""
    gp.loo_log_likelihood(y, quiet=True)
    st = _state(gp)
    got = _batch(gp, vecs, y, kind, quiet)
    _assert_state(gp, st)
    assert _same(got, _loop(gp, vecs, y, kind, quiet)), kind
    return got


KINDS = ["predict", "value", "grad"]


# ---- argument checks, empty batches, no device ---------------------------------------------------------------------

def test_argument_checks_run_before_any_device_call():
    import george_b200 as george
    from george_b200 import kernels
    from george_b200._spec import flatten
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0))
    for fn in (gp.batch_loo_predict, gp.batch_loo_log_likelihood, gp.batch_grad_loo_log_likelihood):
        with pytest.raises(RuntimeError, match="You need to compute the model first"):
            fn(np.zeros((2, len(gp))), np.zeros(3))
    gp._x = np.linspace(0, 1, 5)[:, None]  # what compute() would leave, without touching the device
    gp._yerr2 = np.zeros(5)
    for fn in (gp.batch_loo_predict, gp.batch_loo_log_likelihood, gp.batch_grad_loo_log_likelihood):
        for bad in (np.zeros(len(gp)), np.zeros((2, len(gp) + 1)), np.zeros((1, 2, len(gp)))):
            with pytest.raises(ValueError, match="vectors must have shape"):
                fn(bad, np.zeros(5))
        with pytest.raises(ValueError, match="Dimension mismatch"):
            fn(np.zeros((2, len(gp))), np.zeros(4))

    k = 1.0 * kernels.ExpSquaredKernel(1.0)
    spec, x, ones = flatten(k), np.linspace(0, 1, 5), np.ones((2, 5))
    which = np.ones(len(k), dtype=np.uint32)
    fn = george.BasicSolver.batch_loo_terms
    for w in (None, which):
        with pytest.raises(ValueError, match="params must have shape"):
            fn(spec, np.zeros((2, len(k) + 1)), x, ones, ones, w)
        with pytest.raises(ValueError, match="yerr and r must have shape"):
            fn(spec, np.zeros((2, len(k))), x, np.ones((3, 5)), ones, w)
        with pytest.raises(ValueError, match="x must have shape"):
            fn(spec, np.zeros((2, len(k))), np.zeros((0, 1)), np.ones((2, 0)), np.ones((2, 0)), w)
        with pytest.raises(RuntimeError, match="dimension mismatch"):
            fn(spec, np.zeros((2, len(k))), np.zeros((5, 2)), ones, ones, w)
    with pytest.raises(ValueError, match="which must have shape"):
        fn(spec, np.zeros((2, len(k))), x, ones, ones, which[:1])


def _np65_kernel():
    from george_b200 import kernels
    k = 1.0 * kernels.ExpSquaredKernel(np.eye(8), ndim=8)
    for _ in range(2):
        k = k + 1.0 * kernels.ExpSquaredKernel(np.eye(8), ndim=8)
    assert k.full_size > 64
    return k


def test_more_than_64_parameters_are_rejected_before_any_device_call():
    """Only with which: pass 1 alone has no parameter limit (here it reaches the device check instead)."""
    import george_b200 as george
    from george_b200 import _lib
    from george_b200._spec import flatten
    k = _np65_kernel()
    p = np.tile(k.get_parameter_vector(include_frozen=True), (2, 1))
    args = (flatten(k), p, np.zeros((5, 8)), np.ones((2, 5)), np.ones((2, 5)))
    with pytest.raises(ValueError, match="64"):
        george.BasicSolver.batch_loo_terms(*args, np.ones(k.full_size, dtype=np.uint32))
    if _lib.load().bgp_device_count() == 0:
        with pytest.raises(_lib.BGPError):
            george.BasicSolver.batch_loo_terms(*args)


def test_empty_batch():
    gp, y = _stub_gp()
    e = np.zeros((0, len(gp)))
    mu, var = gp.batch_loo_predict(e, y)
    assert mu.shape == var.shape == (0, N)
    assert gp.batch_loo_log_likelihood(e, y).shape == (0,)
    assert gp.batch_grad_loo_log_likelihood(e, y).shape == (0, len(gp))
    value, grad = gp.batch_grad_loo_log_likelihood(e, y, return_value=True)
    assert value.shape == (0,) and grad.shape == (0, len(gp))
    assert _StubSolver.batch_calls == []
    from george_b200 import BasicSolver, kernels
    from george_b200._spec import flatten
    k = 1.0 * kernels.ExpSquaredKernel(1.0)
    args = (flatten(k), np.zeros((0, len(k))), np.linspace(0, 1, 5), np.ones((0, 5)), np.ones((0, 5)))
    assert [a.shape for a in BasicSolver.batch_loo_terms(*args)] == [(0, 5), (0, 5), (0,)]
    out = BasicSolver.batch_loo_terms(*args, np.ones(len(k), dtype=np.uint32))
    assert [a.shape for a in out] == [(0, 5), (0, 5), (0, 5), (0, len(k)), (0, 5), (0,)]


def test_dense_batch_without_device_raises():
    """No CPU fallback: with valid arguments and no H100, the batched dense path raises BGPError."""
    import george_b200 as george
    from george_b200 import _lib, kernels
    from george_b200._spec import flatten
    if _lib.load().bgp_device_count() > 0:
        pytest.skip("a GPU is present")
    k = 1.0 * kernels.ExpSquaredKernel(1.0)
    with pytest.raises(_lib.BGPError):
        george.BasicSolver.batch_loo_terms(flatten(k), np.zeros((2, len(k))), np.linspace(0, 1, 5), np.ones((2, 5)),
                                           np.ones((2, 5)), np.ones(len(k), dtype=np.uint32))
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0), white_noise=np.log(0.1), fit_white_noise=True)
    gp._x = np.linspace(0, 1, 5)[:, None]
    gp._yerr2 = np.zeros(5)
    for fn in (gp.batch_loo_predict, gp.batch_loo_log_likelihood, gp.batch_grad_loo_log_likelihood):
        with pytest.raises(_lib.BGPError):
            fn(np.zeros((2, len(gp))), np.zeros(5))


# ---- the GP layer around the stub ----------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", KINDS)
def test_stub_matches_the_loop(kind):
    gp, y = _stub_gp()
    vecs = _vectors(gp)
    _check(gp, vecs, y, kind)
    assert len(_StubSolver.batch_calls) == (2 if kind == "grad" else 1)  # (_batch asks the gradient twice)
    for params, r, which in _StubSolver.batch_calls:
        assert params.shape == (5, 2) and r.shape == (5, N)
        assert (which is None) == (kind != "grad")


def test_stub_gradient_layout():
    gp, y = _stub_gp()
    x = gp._x[:, 0]
    vecs = _vectors(gp, nb=3)
    grad = gp.batch_grad_loo_log_likelihood(vecs, y)
    assert np.array_equal(_StubSolver.batch_calls[-1][2], [1, 1])
    for b, v in enumerate(vecs):
        m, c, a, s, lc, lm = v
        wn = a + s * x
        ref = np.concatenate([
            [np.dot(x, BETA * lc), np.sum(BETA * lc)],                          # mean: dmu . beta
            [np.sum(np.exp(wn) * DIAG_A * lm), np.sum(np.exp(wn) * DIAG_A * lm * x)],  # white noise
            [lc, 11.0 * lc],                                                     # kernel: g as given
        ])
        assert np.allclose(grad[b], ref, rtol=1e-13, atol=1e-13), b


def test_stub_frozen_parameters():
    gp, y = _stub_gp(freeze=("kernel:k1:log_constant", "mean:b", "white_noise:s"))
    assert len(gp) == 3
    vecs = _vectors(gp, nb=4)
    _, grad = _check(gp, vecs, y, "grad")
    assert grad.shape == (4, 3)
    assert np.array_equal(_StubSolver.batch_calls[0][2], [0, 1])  # which covers every kernel parameter
    full = _StubSolver.batch_calls[0][0]
    assert np.all(full[:, 0] == np.log(2.0)) and np.array_equal(full[:, 1], vecs[:, 2])


# the member and the full-vector entry that makes it fail, per failure kind (vector: m, b, a, s, log_constant, log_M)
FAILURES = {
    "factorisation": (4, FAIL_LOG_CONSTANT + 1.0),
    "invalid_program": (4, INVALID_LOG_CONSTANT),
    "nan_mean": (1, np.nan),
    "white_noise": (2, NOISE_LIMIT + 1.0),
    "bad_d": (5, -1.5),           # d = D - 1.5: negative from point 0 on
    "mean_gradient": (0, SLOPE_LIMIT + 1.0),
}
# which kinds fail (the value does not look at d's sign beyond -inf, nor at the mean gradient)
FAILS = {"predict": {"factorisation", "invalid_program", "nan_mean", "white_noise"},
         "value": {"factorisation", "invalid_program", "nan_mean", "white_noise"},
         "grad": set(FAILURES)}


def _failing(gp, failure, members=(1, 3)):
    vecs = _vectors(gp, nb=5, seed=6)
    entry, value = FAILURES[failure]
    vecs[list(members), entry] = value
    return vecs


@pytest.mark.parametrize("failure", sorted(FAILURES))
@pytest.mark.parametrize("kind", ["value", "grad"])
def test_quiet_failures_stay_with_their_member(kind, failure):
    gp, y = _stub_gp()
    vecs = _failing(gp, failure)
    got = _check(gp, vecs, y, kind, quiet=True)
    value = got if kind == "value" else got[0]
    fails = failure in FAILS[kind] or (kind == "value" and failure == "bad_d")
    assert np.all(np.isneginf(value[[1, 3]]) == fails), (kind, failure, value)
    assert np.all(np.isfinite(value[[0, 2, 4]]))
    if kind == "grad":
        assert np.all(got[1][[1, 3]] == 0.0) == (failure in FAILS["grad"])
        assert np.all(got[1][[0, 2, 4]] != 0.0)


@pytest.mark.parametrize("failure", sorted(FAILURES))
@pytest.mark.parametrize("kind", KINDS)
def test_first_loop_error_is_raised(kind, failure):
    gp, y = _stub_gp()
    vecs = _failing(gp, failure)
    gp.loo_log_likelihood(y)
    st = _state(gp)
    if failure not in FAILS[kind]:
        got = _batch(gp, vecs, y, kind)
        _assert_state(gp, st)
        assert _same(got, _loop(gp, vecs, y, kind))
        return
    with pytest.raises(Exception) as batch_exc:
        _batch(gp, vecs, y, kind)
    _assert_state(gp, st)
    with pytest.raises(Exception) as loop_exc:
        _loop(gp, vecs, y, kind)
    assert type(batch_exc.value) is type(loop_exc.value)
    assert str(batch_exc.value) == str(loop_exc.value)
    if failure == "bad_d":
        assert str(batch_exc.value) == ("leave-one-out: diag(K^-1) at point 0 is -0.5, not a finite positive number")


def test_the_first_failing_member_decides():
    """Two failure kinds in two members: the one the loop meets first is raised, whatever its kind."""
    gp, y = _stub_gp()
    for order in ((1, 3), (3, 1)):
        vecs = _vectors(gp, nb=5, seed=6)
        vecs[order[0], 1] = np.nan            # NaN mean
        vecs[order[1], 4] = FAIL_LOG_CONSTANT + 1.0  # not positive definite
        for kind in KINDS:
            with pytest.raises(Exception) as batch_exc:
                _batch(gp, vecs, y, kind)
            want = ValueError if order[0] == 1 else LinAlgError
            assert type(batch_exc.value) is want, (order, kind)
            with pytest.raises(want) as loop_exc:
                _loop(gp, vecs, y, kind)
            assert str(batch_exc.value) == str(loop_exc.value)


def test_nonfinite_residual_is_raised_by_the_value_even_when_quiet():
    """A finite mean with a non-finite y: the single value call raises the solver's ValueError under quiet too, the
    gradient absorbs it."""
    gp, y = _stub_gp()
    y = y.copy()
    y[2] = np.inf
    vecs = _vectors(gp, nb=3)
    with pytest.raises(ValueError) as batch_exc:
        gp.batch_loo_log_likelihood(vecs, y, quiet=True)
    with pytest.raises(ValueError) as loop_exc:
        _loop(gp, vecs, y, "value", quiet=True)
    assert str(batch_exc.value) == str(loop_exc.value)
    got = gp.batch_grad_loo_log_likelihood(vecs, y, quiet=True, return_value=True)
    assert np.all(np.isneginf(got[0])) and np.all(got[1] == 0.0)


# ---- solvers and kernels that take the loop ------------------------------------------------------------------------

def _trivial_gp():
    import george_b200 as george
    x, yerr, y = _data()
    gp = george.GP(mean=_line_mean(0.3, -0.1), fit_mean=True, white_noise=_log_linear_noise(-2.0, 0.1),
                   fit_white_noise=True)
    assert gp.solver_type is george.TrivialSolver
    gp.compute(x, yerr)
    return gp, y


@pytest.mark.parametrize("kind", KINDS)
def test_trivial_solver_takes_the_loop(kind):
    import george_b200 as george
    assert getattr(george.TrivialSolver, "batch_loo_terms", None) is None
    gp, y = _trivial_gp()
    vecs = _vectors(gp)
    _check(gp, vecs, y, kind)
    vecs[2, 1] = np.nan
    if kind != "predict":
        got = _check(gp, vecs, y, kind, quiet=True)
        assert np.isneginf(got[2] if kind == "value" else got[0][2])
    with pytest.raises(ValueError, match="mean function"):
        _batch(gp, vecs, y, kind)


@pytest.mark.parametrize("kind", KINDS)
def test_hodlr_typed_gp_takes_the_loop(kind):
    import george_b200 as george
    assert george.HODLRSolver.batch_loo_terms is None

    class StubHODLR(george.HODLRSolver):
        __init__ = _StubSolver.__init__
        compute = _StubSolver.compute
        dot_solve = _StubSolver.dot_solve
        loo_terms = _StubSolver.loo_terms

    gp, y = _stub_gp(solver=StubHODLR)
    _check(gp, _vectors(gp), y, kind)
    assert _StubSolver.batch_calls == []


def test_more_than_64_kernel_parameters_take_the_loop_for_the_gradient():
    """The gradient takes the loop (whose single call raises the device's "64" error; here the stub's loo_terms
    answers); the value and the predictive still run batched."""
    import george_b200 as george
    gp = george.GP(_np65_kernel(), mean=0.1, fit_mean=True, white_noise=np.log(0.01), fit_white_noise=True,
                   solver=_StubSolver)
    rng = np.random.default_rng(8)
    gp.compute(rng.uniform(0, 1, (N, 8)), 0.1)
    y = rng.standard_normal(N)
    _StubSolver.batch_calls = []
    vecs = _vectors(gp, nb=3)
    _check(gp, vecs, y, "grad")
    assert _StubSolver.batch_calls == []
    _check(gp, vecs, y, "value")
    _check(gp, vecs, y, "predict")
    assert len(_StubSolver.batch_calls) == 2
