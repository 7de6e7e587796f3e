# -*- coding: utf-8 -*-
"""GP.batch_fisher_information on the host (no GPU).

* the argument checks that run before any device call, the empty results, the error raised without a device;
* the GP layer around a stub solver whose ``batch_fisher_terms``, ``fisher_terms`` and ``apply_inverse`` return fixed
  arrays, a function of the member's kernel parameters, white-noise vectors, mean gradients and residual: the layout
  with frozen parameters, a fitted line mean and a log-linear white noise, ``quiet`` member by member for every
  failure kind, the first loop error, the GP's state, and the ``NotImplementedError`` of a HODLR-typed GP;
* the per-vector loop taken by ``TrivialSolver``, by more than 64 kernel parameters and by a GP whose only active
  parameters are the mean's.
"""
import numpy as np
import pytest
from numpy.linalg import LinAlgError

from test_batch_loo_host import (ALPHA, DIAG_A, D, FAIL_LOG_CONSTANT, INVALID_LOG_CONSTANT, N, NOISE_LIMIT,
                                 SLOPE_LIMIT, _assert_state, _data, _info, _np65_kernel, _state, _vectors)

NOISE_SLOPE_LIMIT = 10.0  # white noise "s" above it: its gradient raises ValueError; below minus it, RuntimeError


def _line_mean(m, b):
    """A line whose gradient is NaN for m > SLOPE_LIMIT and, for m < -SLOPE_LIMIT, finite in longdouble but infinite
    once converted to float64 (the solve's check then raises)."""
    from george_b200.modeling import Model

    class LineMean(Model):
        parameter_names = ("m", "b")

        def get_value(self, x):
            return self.m * np.asarray(x).flatten() + self.b

        def compute_gradient(self, x):
            x = np.asarray(x).flatten()
            g = np.vstack([x, np.ones_like(x)])
            if self.m > SLOPE_LIMIT:
                return g * np.nan
            if self.m < -SLOPE_LIMIT:
                return g.astype(np.longdouble) * np.longdouble(1e300) * np.longdouble(1e300)
            return g

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
            if self.s > NOISE_SLOPE_LIMIT:
                raise ValueError("white-noise gradient out of range")
            if self.s < -NOISE_SLOPE_LIMIT:
                raise RuntimeError("white-noise gradient failed")
            x = np.asarray(x).flatten()
            return np.vstack([np.ones_like(x), x])

    return LogLinearNoise(a=a, s=s)


def _rows(kp, which, v):
    """The stub's Fisher rows of one member: kernel parameters ``kp``, white-noise vectors ``v`` ``(nv, N)``."""
    which = np.asarray(which)
    nrow = int(np.count_nonzero(which)) + len(v)
    k = np.arange(1.0, nrow + 1)
    rows = np.outer(k, 10.0 * np.arange(len(which)) + 1.0) * kp[0] * (which != 0)
    rdiag = np.outer(k, D * kp[1])
    rdiag[nrow - len(v):] += np.asarray(v) * kp[0]
    return rows, rdiag


def _grad_terms(kp, r, which):
    g = (10.0 * np.arange(len(which)) + 1.0) * kp[0] * (np.asarray(which) != 0)
    return ALPHA * kp[0] + r, g, DIAG_A * kp[1]


def _solve(kp, b):
    """The stub's K^-1 b, with BasicSolver.apply_inverse's layout and right-hand side check."""
    from george_b200.solvers.basic import _check_finite
    b = np.array(b, dtype=np.float64, order="F")
    _check_finite(b)
    b *= (D * kp[1]).reshape((-1,) + (1,) * (b.ndim - 1))
    return b


class _StubSolver(object):
    """fisher_terms, apply_inverse and batch_fisher_terms from _rows, _grad_terms and _solve; compute fails as the
    batch's info says."""

    batch_calls = []

    def __init__(self, kernel, **kwargs):
        self.kernel = kernel
        self.computed = False

    def _kp(self):
        return self.kernel.get_parameter_vector(include_frozen=True)

    def compute(self, x, yerr):
        info = _info(self._kp())
        if info > 0:
            raise LinAlgError("%d-th leading minor of the array is not positive definite" % info)
        if info < 0:
            raise ValueError("invalid kernel")
        self.log_determinant = 0.0
        self.computed = True

    def apply_inverse(self, y, in_place=False):
        return _solve(self._kp(), y)

    def dot_solve(self, y):
        return 0.0

    def fisher_terms(self, r, which, v):
        from george_b200.solvers.basic import NONFINITE_RHS
        if r is not None and not np.all(np.isfinite(r)):
            raise ValueError(NONFINITE_RHS)
        terms = None if r is None else _grad_terms(self._kp(), np.asarray(r), which)
        return (terms,) + _rows(self._kp(), which, v)

    @staticmethod
    def batch_fisher_terms(spec, params, x, yerr, r, which, v, dmu):
        _StubSolver.batch_calls.append((np.array(params), None if r is None else np.array(r), np.array(which),
                                        np.array(v), np.array(dmu)))
        nb = len(params)
        rows = np.stack([_rows(params[b], which, v[b])[0] for b in range(nb)])
        rdiag = np.stack([_rows(params[b], which, v[b])[1] for b in range(nb)])
        kdmu = np.stack([_solve(params[b], dmu[b].T).T for b in range(nb)])
        info = np.array([_info(p) for p in params], dtype=np.int32)
        terms = None
        if r is not None:
            t = [_grad_terms(params[b], r[b], which) for b in range(nb)]
            terms = tuple(np.stack([tb[k] for tb in t]) for k in range(3))
        for a in (rows, rdiag, kdmu) + (terms or ()):
            a[info != 0] = np.nan
        return terms, rows, rdiag, kdmu, info


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


def _loop(gp, vecs, y, quiet=False):
    p0 = gp.get_parameter_vector()
    res = []
    try:
        for v in vecs:
            gp.set_parameter_vector(v)
            res.append(gp.fisher_information(y, quiet=quiet))
    finally:
        gp.set_parameter_vector(p0)
    if y is None:
        return np.stack(res)
    return np.stack([r[0] for r in res]), np.stack([r[1] for r in res])


def _same(got, want):
    if isinstance(want, tuple):
        return all(_same(a, b) for a, b in zip(got, want))
    return got.shape == want.shape and np.array_equal(got, want, equal_nan=True)


def _check(gp, vecs, y, quiet=False):
    """batch == loop bit for bit, the GP left as it was; returns the batch's result."""
    gp.fisher_information(quiet=True)
    st = _state(gp)
    got = gp.batch_fisher_information(vecs, y, quiet=quiet)
    _assert_state(gp, st)
    assert _same(got, _loop(gp, vecs, y, quiet))
    return got


# ---- argument checks, empty batches, no device ---------------------------------------------------------------------

def test_argument_checks_run_before_any_device_call():
    import george_b200 as george
    from george_b200 import kernels
    from george_b200._spec import flatten
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0))
    with pytest.raises(RuntimeError, match="You need to compute the model first"):
        gp.batch_fisher_information(np.zeros((2, len(gp))))
    gp._x = np.linspace(0, 1, 5)[:, None]  # what compute() would leave, without touching the device
    gp._yerr2 = np.zeros(5)
    for bad in (np.zeros(len(gp)), np.zeros((2, len(gp) + 1)), np.zeros((1, 2, len(gp)))):
        with pytest.raises(ValueError, match="vectors must have shape"):
            gp.batch_fisher_information(bad)
    with pytest.raises(ValueError, match="Dimension mismatch"):
        gp.batch_fisher_information(np.zeros((2, len(gp))), np.zeros(4))

    k = 1.0 * kernels.ExpSquaredKernel(1.0)
    spec, x, ones = flatten(k), np.linspace(0, 1, 5), np.ones((2, 5))
    which = np.ones(len(k), dtype=np.uint32)
    v, dmu = np.ones((2, 1, 5)), np.ones((2, 0, 5))
    fn = george.BasicSolver.batch_fisher_terms
    for r in (None, ones):
        with pytest.raises(ValueError, match="params must have shape"):
            fn(spec, np.zeros((2, len(k) + 1)), x, ones, r, which, v, dmu)
        with pytest.raises(ValueError, match="yerr and r must have shape"):
            fn(spec, np.zeros((2, len(k))), x, np.ones((3, 5)), r, which, v, dmu)
        with pytest.raises(ValueError, match="which must have shape"):
            fn(spec, np.zeros((2, len(k))), x, ones, r, which[:1], v, dmu)
        for bv, bd in ((np.ones((2, 5)), dmu), (np.ones((3, 1, 5)), dmu), (v, np.ones((2, 1, 4)))):
            with pytest.raises(ValueError, match="v and dmu must have shape"):
                fn(spec, np.zeros((2, len(k))), x, ones, r, which, bv, bd)
        with pytest.raises(RuntimeError, match="dimension mismatch"):
            fn(spec, np.zeros((2, len(k))), np.zeros((5, 2)), ones, r, which, v, dmu)
    with pytest.raises(ValueError, match="yerr and r must have shape"):
        fn(spec, np.zeros((2, len(k))), x, ones, np.ones((2, 4)), which, v, dmu)


def test_more_than_64_parameters_are_rejected_before_any_device_call():
    import george_b200 as george
    from george_b200._spec import flatten
    k = _np65_kernel()
    p = np.tile(k.get_parameter_vector(include_frozen=True), (2, 1))
    with pytest.raises(ValueError, match="64"):
        george.BasicSolver.batch_fisher_terms(flatten(k), p, np.zeros((5, 8)), np.ones((2, 5)), None,
                                              np.ones(k.full_size, dtype=np.uint32), np.ones((2, 0, 5)),
                                              np.ones((2, 0, 5)))


def test_empty_batch():
    gp, y = _stub_gp()
    e = np.zeros((0, len(gp)))
    assert gp.batch_fisher_information(e).shape == (0, len(gp), len(gp))
    grad, F = gp.batch_fisher_information(e, y)
    assert grad.shape == (0, len(gp)) and F.shape == (0, len(gp), len(gp))
    assert _StubSolver.batch_calls == []
    from george_b200 import BasicSolver, kernels
    from george_b200._spec import flatten
    k = 1.0 * kernels.ExpSquaredKernel(1.0)
    which = np.array([1, 0], dtype=np.uint32)
    args = (flatten(k), np.zeros((0, len(k))), np.linspace(0, 1, 5), np.ones((0, 5)))
    terms, rows, rdiag, kdmu, info = BasicSolver.batch_fisher_terms(*args, None, which, np.ones((0, 2, 5)),
                                                                   np.ones((0, 3, 5)))
    assert terms is None
    assert [a.shape for a in (rows, rdiag, kdmu, info)] == [(0, 3, 2), (0, 3, 5), (0, 3, 5), (0,)]
    terms, *_ = BasicSolver.batch_fisher_terms(*args, np.ones((0, 5)), which, np.ones((0, 2, 5)), np.ones((0, 3, 5)))
    assert [a.shape for a in terms] == [(0, 5), (0, 2), (0, 5)]


def test_dense_batch_without_device_raises():
    """No CPU fallback: with valid arguments and no H100, the batched dense path raises BGPError."""
    import george_b200 as george
    from george_b200 import _lib, kernels
    from george_b200._spec import flatten
    if _lib.load().bgp_device_count() > 0:
        pytest.skip("a GPU is present")
    k = 1.0 * kernels.ExpSquaredKernel(1.0)
    with pytest.raises(_lib.BGPError):
        george.BasicSolver.batch_fisher_terms(flatten(k), np.zeros((2, len(k))), np.linspace(0, 1, 5),
                                              np.ones((2, 5)), None, np.ones(len(k), dtype=np.uint32),
                                              np.ones((2, 1, 5)), np.ones((2, 0, 5)))
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0), white_noise=np.log(0.1), fit_white_noise=True)
    gp._x = np.linspace(0, 1, 5)[:, None]
    gp._yerr2 = np.zeros(5)
    for y in (None, np.zeros(5)):
        with pytest.raises(_lib.BGPError):
            gp.batch_fisher_information(np.zeros((2, len(gp))), y)


# ---- the GP layer around the stub ----------------------------------------------------------------------------------

@pytest.mark.parametrize("with_y", [False, True])
def test_stub_matches_the_loop(with_y):
    gp, y = _stub_gp()
    vecs = _vectors(gp)
    _check(gp, vecs, y if with_y else None)
    assert len(_StubSolver.batch_calls) == 1
    params, r, which, v, dmu = _StubSolver.batch_calls[0]
    assert params.shape == (5, 2) and (r is None) != with_y and np.array_equal(which, [1, 1])
    assert v.shape == (5, 2, N) and dmu.shape == (5, 2, N)
    if with_y:
        assert r.shape == (5, N)


def test_stub_layout():
    gp, y = _stub_gp()
    x = gp._x[:, 0]
    vecs = _vectors(gp, nb=3)
    grad, F = gp.batch_fisher_information(vecs, y)
    for b, vec in enumerate(vecs):
        m, c, a, s, lc, lm = vec
        dmu = np.vstack([x, np.ones_like(x)])
        v = np.exp(a + s * x)[None, :] * np.vstack([np.ones_like(x), x])
        rows, rdiag = _rows([lc, lm], [1, 1], v)
        M = dmu.dot(_solve([lc, lm], dmu.T))
        R = np.zeros((4, 4))
        order = [2, 3, 0, 1]  # white noise first, then kernel
        R[:, :2] = 0.5 * rdiag[order].dot(v.T)
        R[:, 2:] = 0.5 * rows[order]
        want = np.zeros((6, 6))
        want[:2, :2] = 0.5 * (M + M.T)
        want[2:, 2:] = 0.5 * (R + R.T)
        assert np.allclose(F[b], want, rtol=1e-13, atol=0), b
        assert np.array_equal(F[b], F[b].T)
        alpha, g, diag = _grad_terms([lc, lm], y - (m * x + c), [1, 1])
        want_g = np.concatenate([dmu.dot(alpha), 0.5 * (np.exp(a + s * x) * diag).dot(np.vstack([np.ones_like(x), x]).T),
                                 0.5 * g])
        assert np.allclose(grad[b], want_g, rtol=1e-12, atol=1e-12), b


def test_stub_frozen_parameters():
    gp, y = _stub_gp(freeze=("kernel:k1:log_constant", "mean:b", "white_noise:s"))
    assert len(gp) == 3
    vecs = _vectors(gp, nb=4)
    for yy in (None, y):
        got = _check(gp, vecs, yy)
        assert (got if yy is None else got[1]).shape == (4, 3, 3)
    params, _, which, v, dmu = _StubSolver.batch_calls[0]
    assert np.array_equal(which, [0, 1])  # which covers every kernel parameter
    assert v.shape == (4, 1, N) and dmu.shape == (4, 1, N)
    assert np.all(params[:, 0] == np.log(2.0)) and np.array_equal(params[:, 1], vecs[:, 2])


# the member and the full-vector entry that makes it fail, per failure kind (vector: m, b, a, s, log_constant, log_M)
FAILURES = {
    "factorisation": (4, FAIL_LOG_CONSTANT + 1.0),
    "invalid_program": (4, INVALID_LOG_CONSTANT),
    "white_noise": (2, NOISE_LIMIT + 1.0),
    "nan_mean": (1, np.nan),                      # with y the residual fails, without y the mean gradient
    "white_noise_gradient": (3, NOISE_SLOPE_LIMIT + 1.0),
    "white_noise_gradient_runtime": (3, -NOISE_SLOPE_LIMIT - 1.0),  # not a ValueError: quiet does not absorb it
    "mean_gradient": (0, SLOPE_LIMIT + 1.0),
    "mean_gradient_overflow": (0, -SLOPE_LIMIT - 1.0),  # the solve's non-finite right-hand side
}
NOT_ABSORBED = {"white_noise_gradient_runtime"}


def _fails(failure, y):
    """Whether the failure reaches the single call: without y no residual is formed, and a NaN slope leaves the
    line's gradient finite."""
    return not (failure == "nan_mean" and y is None)


def _failing(gp, failure, members=(1, 3)):
    vecs = _vectors(gp, nb=5, seed=6)
    entry, value = FAILURES[failure]
    vecs[list(members), entry] = value
    return vecs


@pytest.mark.parametrize("failure", sorted(FAILURES))
@pytest.mark.parametrize("with_y", [False, True])
def test_quiet_failures_stay_with_their_member(failure, with_y):
    gp, y = _stub_gp()
    y = y if with_y else None
    vecs = _failing(gp, failure)
    if failure in NOT_ABSORBED:
        with pytest.raises(RuntimeError, match="white-noise gradient failed"):
            gp.batch_fisher_information(vecs, y, quiet=True)
        return
    with np.errstate(over="ignore"):
        got = _check(gp, vecs, y, quiet=True)
    F = got if y is None else got[1]
    assert np.all(F[[1, 3]] == 0.0) == _fails(failure, y)
    assert np.all(F[[0, 2, 4]].any(axis=(1, 2)))
    if y is not None:
        assert np.all(got[0][[1, 3]] == 0.0) and np.all(got[0][[0, 2, 4]].any(axis=1))


@pytest.mark.parametrize("failure", sorted(FAILURES))
@pytest.mark.parametrize("with_y", [False, True])
def test_first_loop_error_is_raised(failure, with_y):
    gp, y = _stub_gp()
    y = y if with_y else None
    vecs = _failing(gp, failure)
    gp.fisher_information()
    st = _state(gp)
    if not _fails(failure, y):
        _check(gp, vecs, y)
        return
    with np.errstate(over="ignore"):
        with pytest.raises(Exception) as batch_exc:
            gp.batch_fisher_information(vecs, y)
        _assert_state(gp, st)
        with pytest.raises(Exception) as loop_exc:
            _loop(gp, vecs, y)
    assert type(batch_exc.value) is type(loop_exc.value)
    assert str(batch_exc.value) == str(loop_exc.value)


def test_the_first_failing_member_decides():
    """Two failure kinds in two members: the one the loop meets first is raised, whatever its kind."""
    gp, y = _stub_gp()
    for order in ((1, 3), (3, 1)):
        vecs = _vectors(gp, nb=5, seed=6)
        vecs[order[0], 3] = NOISE_SLOPE_LIMIT + 1.0   # the white-noise gradient
        vecs[order[1], 4] = FAIL_LOG_CONSTANT + 1.0   # not positive definite
        for yy in (None, y):
            with pytest.raises(Exception) as batch_exc:
                gp.batch_fisher_information(vecs, yy)
            want = ValueError if order[0] == 1 else LinAlgError
            assert type(batch_exc.value) is want, (order, yy is None)
            with pytest.raises(want) as loop_exc:
                _loop(gp, vecs, yy)
            assert str(batch_exc.value) == str(loop_exc.value)


def test_nonfinite_residual_is_absorbed_when_quiet():
    gp, y = _stub_gp()
    y = y.copy()
    y[2] = np.inf
    vecs = _vectors(gp, nb=3)
    grad, F = _check(gp, vecs, y, quiet=True)
    assert np.all(grad == 0.0) and np.all(F == 0.0)
    with pytest.raises(ValueError) as batch_exc:
        gp.batch_fisher_information(vecs, y)
    with pytest.raises(ValueError) as loop_exc:
        _loop(gp, vecs, y)
    assert str(batch_exc.value) == str(loop_exc.value)
    _check(gp, vecs, None)  # without y the residual is never formed


def test_hodlr_typed_gp_raises_before_any_work():
    import george_b200 as george
    from george_b200.solvers.hodlr import FISHER_HODLR
    assert george.HODLRSolver.batch_fisher_terms is None

    class StubHODLR(george.HODLRSolver):
        __init__ = _StubSolver.__init__
        _kp = _StubSolver._kp
        compute = _StubSolver.compute

    gp, y = _stub_gp(solver=StubHODLR)
    st = _state(gp)
    for yy in (None, y):
        for vecs in (_vectors(gp), np.zeros((0, len(gp))), np.zeros(3)):
            with pytest.raises(NotImplementedError) as exc:
                gp.batch_fisher_information(vecs, yy)
            assert str(exc.value) == FISHER_HODLR
    _assert_state(gp, st)
    assert _StubSolver.batch_calls == []


# ---- solvers and GPs that take the loop ----------------------------------------------------------------------------

def test_trivial_solver_takes_the_loop():
    import george_b200 as george
    assert getattr(george.TrivialSolver, "batch_fisher_terms", None) is None
    x, yerr, y = _data()
    # without y and a fitted mean: the single call would need TrivialSolver.get_inverse (with y) and its
    # apply_inverse of several columns (a fitted mean), which it does not have
    gp = george.GP(mean=0.1, white_noise=_log_linear_noise(-2.0, 0.1), fit_white_noise=True)
    assert gp.solver_type is george.TrivialSolver
    gp.compute(x, yerr)
    vecs = _vectors(gp)
    _check(gp, vecs, None)
    vecs[2, 0] = NOISE_LIMIT + 1.0
    got = _check(gp, vecs, None, quiet=True)
    assert np.all(got[2] == 0.0) and np.all(np.delete(got, 2, axis=0) != 0.0)
    with pytest.raises(ValueError, match="white noise out of range"):
        gp.batch_fisher_information(vecs)


def test_more_than_64_kernel_parameters_take_the_loop():
    """The loop's single call raises the device's "64" error; here the stub's fisher_terms answers."""
    import george_b200 as george
    gp = george.GP(_np65_kernel(), mean=0.1, fit_mean=True, white_noise=np.log(0.01), fit_white_noise=True,
                   solver=_StubSolver)
    rng = np.random.default_rng(8)
    gp.compute(rng.uniform(0, 1, (N, 8)), 0.1)
    y = rng.standard_normal(N)
    _StubSolver.batch_calls = []
    vecs = _vectors(gp, nb=3)
    for yy in (None, y):
        _check(gp, vecs, yy)
    assert _StubSolver.batch_calls == []


def test_mean_only_gp_takes_the_loop():
    gp, y = _stub_gp(freeze=("kernel:k1:log_constant", "kernel:k2:metric:log_M_0_0", "white_noise:a",
                             "white_noise:s"))
    assert len(gp) == 2
    vecs = _vectors(gp, nb=3)
    for yy in (None, y):
        got = _check(gp, vecs, yy)
        assert np.all((got if yy is None else got[1])[:, 0, 0] > 0)
    assert _StubSolver.batch_calls == []
