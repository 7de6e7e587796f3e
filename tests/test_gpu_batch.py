# -*- coding: utf-8 -*-
"""GP.batch_log_likelihood / BasicSolver.batch_log_likelihood on the device: every member's log-determinant is the
single-matrix path's bit for bit, its solve agrees with dot_solve, failures stay with their member, the results do not
depend on B, the position or the chunking, and the launch count does not grow with B."""
import pickle

import numpy as np
import pytest

import hiprec

pytestmark = pytest.mark.gpu

LOGDET_TOL = 5e-14      # |logdet - ref| / max(1, |ref|)   (the bars of tests/test_gpu_dense_blocks.py)
DOT_TOL = 5e-13         # |r^T K^-1 r - ref| / |ref|, cond(K) <~ 1e4
SIZES = [1, 2, 63, 64, 65, 129, 300, 1000, 2049]


def _zoo():
    from george_b200 import kernels as K
    return [
        ("expsq_1d", 1.0 * K.ExpSquaredKernel(1.0), 1),
        ("m52_3d_iso", K.Matern52Kernel(0.5, ndim=3), 3),
        ("m52_3d_axis", 1.3 * K.Matern52Kernel([0.5, 1.0, 2.0], ndim=3), 3),
        ("expsq_3d_general", K.ExpSquaredKernel([[1.0, 0.1, 0.2], [0.1, 2.0, 0.3], [0.2, 0.3, 1.5]], ndim=3), 3),
        ("sum_expsq_expsine2", 1.0 * K.ExpSquaredKernel(1.0, ndim=3)
         + 0.5 * K.ExpSine2Kernel(gamma=1.0, log_period=np.log(3.0), ndim=3, axes=1), 3),
        ("expsq_block", K.ExpSquaredKernel(1.0, ndim=3, block=[(-0.5, 0.5)] * 3), 3),
        ("user_cauchy", 0.8 * K.CauchyKernel(metric=0.7, ndim=2), 2),
    ]


def _inputs(n, ndim, nb, seed):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-2, 2, (n, ndim))
    sig = 0.5 + 0.5 * rng.uniform(size=(nb, n))
    r = rng.standard_normal((nb, n))
    return x, sig, r


def _perturbed(kernel, nb, seed, scale=0.05):
    rng = np.random.default_rng(seed)
    p0 = kernel.get_parameter_vector(include_frozen=True)
    return p0 + scale * rng.standard_normal((nb, len(p0)))


def _single(kernel, p, x, sig, r):
    from george_b200 import BasicSolver
    p0 = kernel.get_parameter_vector(include_frozen=True)
    kernel.set_parameter_vector(p, include_frozen=True)
    try:
        s = BasicSolver(kernel)
        s.compute(x, sig)
        return s.log_determinant, s.dot_solve(r)
    finally:
        kernel.set_parameter_vector(p0, include_frozen=True)


@pytest.mark.parametrize("name", [z[0] for z in _zoo()])
def test_members_match_the_single_path(gpu, name):
    from george_b200 import BasicSolver
    from george_b200._spec import flatten
    _, kernel, ndim = [z for z in _zoo() if z[0] == name][0]
    for n in SIZES:
        params = _perturbed(kernel, 7, n)
        x, sig, r = _inputs(n, ndim, 7, n + 1)
        ld, q, info = BasicSolver.batch_log_likelihood(flatten(kernel), params, x, sig, r)
        assert np.all(info == 0), (name, n, info)
        for b in range(7):
            ld1, q1 = _single(kernel, params[b], x, sig[b], r[b])
            assert ld[b] == ld1, (name, n, b, ld[b], ld1)
            assert abs(q[b] - q1) <= 1e-13 * abs(q1), (name, n, b, q[b], q1)


@pytest.mark.parametrize("n", [63, 65, 300, 700])
def test_accuracy_against_extended_precision(gpu, n):
    from george_b200 import BasicSolver, kernels
    from george_b200._spec import flatten
    kernel = 1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3)
    params = _perturbed(kernel, 5, 7 * n)
    x, sig, r = _inputs(n, 3, 5, n)
    ld, q, info = BasicSolver.batch_log_likelihood(flatten(kernel), params, x, sig, r)
    assert np.all(info == 0)
    p0 = kernel.get_parameter_vector(include_frozen=True)
    try:
        for b in range(3):
            kernel.set_parameter_vector(params[b], include_frozen=True)
            K = kernel.get_value(x)
            K[np.diag_indices(n)] += sig[b] * sig[b]
            assert np.linalg.cond(K) < 1e4
            L = hiprec.chol_ld(K)
            ref_ld = hiprec.logdet_ld(L)
            ref_q = float(np.dot(r[b].astype(hiprec.LD), hiprec.solve_ld(L, r[b])))
            assert abs(float(ld[b] - ref_ld)) / max(1.0, abs(float(ref_ld))) <= LOGDET_TOL
            assert abs(q[b] - ref_q) / abs(ref_q) <= DOT_TOL
    finally:
        kernel.set_parameter_vector(p0, include_frozen=True)


def _co2_gp(n=500, seed=0):
    """The hyper-parameter tutorial's GP: the CO2 kernel (a sum of four products), a fitted constant mean and a
    fitted white noise, yerr = 0."""
    import george_b200 as george
    from george_b200 import kernels
    k1 = 66 ** 2 * kernels.ExpSquaredKernel(metric=67 ** 2)
    k2 = 2.4 ** 2 * kernels.ExpSquaredKernel(90 ** 2) * kernels.ExpSine2Kernel(gamma=2 / 1.3 ** 2, log_period=0.0)
    k3 = 0.66 ** 2 * kernels.RationalQuadraticKernel(log_alpha=np.log(0.78), metric=1.2 ** 2)
    k4 = 0.18 ** 2 * kernels.ExpSquaredKernel(1.6 ** 2)
    rng = np.random.default_rng(seed)
    t = np.sort(rng.uniform(1958, 2003, n))
    y = 315 + 1.3 * (t - 1958) + 3 * np.sin(2 * np.pi * t) + 0.3 * rng.standard_normal(n)
    gp = george.GP(k1 + k2 + k3 + k4, mean=np.mean(y), fit_mean=True, white_noise=np.log(0.19 ** 2),
                   fit_white_noise=True)
    gp.compute(t)
    return gp, y


def _state(gp):
    return (gp.get_parameter_vector(include_frozen=True).copy(), gp.computed, gp.solver, gp._alpha, gp._y,
            gp.kernel.dirty)


def _assert_state(gp, st):
    now = _state(gp)
    assert np.array_equal(st[0], now[0])
    assert now[1] == st[1] and now[5] == st[5]
    assert now[2] is st[2] and now[3] is st[3] and now[4] is st[4]


def _loop(gp, vecs, y, quiet):
    p0 = gp.get_parameter_vector()
    out = np.empty(len(vecs))
    try:
        for b, v in enumerate(vecs):
            gp.set_parameter_vector(v)
            out[b] = gp.log_likelihood(y, quiet=quiet)
    finally:
        gp.set_parameter_vector(p0)
    return out


def _close(a, b):
    return np.all(np.abs(a - b) <= 1e-12 * np.maximum(1.0, np.abs(b)))


def test_emcee_step_co2(gpu):
    gp, y = _co2_gp()
    ll0 = gp.log_likelihood(y)
    rng = np.random.default_rng(5)
    vecs = gp.get_parameter_vector() + 1e-4 * rng.standard_normal((36, len(gp)))
    st = _state(gp)
    got = gp.batch_log_likelihood(vecs, y, quiet=True)
    _assert_state(gp, st)
    assert gp.log_likelihood(y) == ll0  # no refactorisation, the same cached result
    assert gp.solver is st[2]
    want = _loop(gp, vecs, y, True)
    assert np.all(np.isfinite(got)) and _close(got, want), np.max(np.abs(got - want))


def test_non_constant_mean_with_frozen_parameters(gpu):
    """A polynomial mean model (the model-fitting tutorial's ``PolynomialModel``, restated) with one parameter
    frozen: the members' residuals come from the model evaluated at each member's parameters."""
    import george_b200 as george
    from george_b200 import kernels
    from george_b200.modeling import Model

    class PolynomialModel(Model):
        parameter_names = ("m", "b")

        def get_value(self, t):
            t = t.flatten()
            return t * self.m + self.b

    rng = np.random.default_rng(6)
    t = np.sort(rng.uniform(-5, 5, 300))
    y = 0.5 * t - 0.2 + np.sin(t) + 0.1 * rng.standard_normal(300)
    mean = PolynomialModel(m=0.4, b=0.0)
    gp = george.GP(0.5 * kernels.Matern32Kernel(1.5), mean=mean, white_noise=np.log(0.1 ** 2), fit_white_noise=True)
    gp.freeze_parameter("mean:b")
    gp.compute(t, 0.05)
    gp.log_likelihood(y)
    vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((9, len(gp)))
    st = _state(gp)
    got = gp.batch_log_likelihood(vecs, y)
    _assert_state(gp, st)
    assert np.array_equal(gp.mean.get_parameter_vector(include_frozen=True), [0.4, 0.0])
    assert _close(got, _loop(gp, vecs, y, False))


def _dot_gp():
    import george_b200 as george
    from george_b200 import kernels
    x = np.linspace(0.1, 1, 50)
    gp = george.GP(kernels.DotProductKernel(), white_noise=np.log(0.1), fit_white_noise=True)
    gp.compute(x, 0.0)
    y = np.cos(x)
    return gp, y


def test_failures_stay_with_their_member(gpu):
    from george_b200 import BasicSolver
    gp, y = _dot_gp()
    gp.log_likelihood(y)
    vecs = np.full((8, len(gp)), np.log(0.1))
    bad = [2, 5]
    vecs[bad, 0] = -80.0  # K = x x^T + 1.8e-35 I: rank one, not positive definite
    st = _state(gp)
    got = gp.batch_log_likelihood(vecs, y, quiet=True)
    _assert_state(gp, st)
    want = _loop(gp, vecs, y, True)
    assert np.all(np.isneginf(got[bad]))
    good = [b for b in range(8) if b not in bad]
    assert np.all(np.isfinite(got[good])) and _close(got[good], want[good])

    gp.log_likelihood(y)  # (the reference loop above left the GP at another factorisation)
    st = _state(gp)
    with pytest.raises(np.linalg.LinAlgError) as batch_exc:
        gp.batch_log_likelihood(vecs, y, quiet=False)
    _assert_state(gp, st)
    with pytest.raises(np.linalg.LinAlgError) as loop_exc:
        _loop(gp, vecs, y, False)
    assert str(batch_exc.value) == str(loop_exc.value)

    # info: the leading-minor index the single path reports
    from george_b200._spec import flatten
    x = gp._x
    sig = np.sqrt(np.zeros((8, 50)) + np.exp(vecs[:, :1]))
    _, _, info = BasicSolver.batch_log_likelihood(flatten(gp.kernel), np.zeros((8, 0)), x, sig, np.ones((8, 50)))
    for b in range(8):
        if b in bad:
            with pytest.raises(np.linalg.LinAlgError) as e:
                BasicSolver(gp.kernel).compute(x, sig[b])
            assert info[b] > 0 and str(e.value).startswith("%d-th" % info[b])
        else:
            assert info[b] == 0


def test_results_do_not_depend_on_batch_position_or_chunking(gpu, monkeypatch):
    from george_b200 import BasicSolver, kernels
    from george_b200._spec import flatten
    kernel = 1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3)
    spec = flatten(kernel)
    n = 130
    params = _perturbed(kernel, 64, 11)
    x, sig, r = _inputs(n, 3, 64, 12)
    monkeypatch.delenv("BGP_BATCH_CHUNK", raising=False)
    ld, q, _ = BasicSolver.batch_log_likelihood(spec, params, x, sig, r)
    ld2, q2, _ = BasicSolver.batch_log_likelihood(spec, params, x, sig, r)
    assert np.array_equal(ld, ld2) and np.array_equal(q, q2)
    for b in (0, 17, 63):
        l1, q1, _ = BasicSolver.batch_log_likelihood(spec, params[b:b + 1], x, sig[b:b + 1], r[b:b + 1])
        assert l1[0] == ld[b] and q1[0] == q[b]
    # member 17 at the last position
    order = [i for i in range(64) if i != 17] + [17]
    l3, q3, _ = BasicSolver.batch_log_likelihood(spec, params[order], x, sig[order], r[order])
    assert l3[-1] == ld[17] and q3[-1] == q[17]
    for chunk in ("1", "5", "64"):
        monkeypatch.setenv("BGP_BATCH_CHUNK", chunk)
        lc, qc, _ = BasicSolver.batch_log_likelihood(spec, params, x, sig, r)
        assert np.array_equal(lc, ld) and np.array_equal(qc, q), chunk


def test_launch_count_does_not_grow_with_the_batch(gpu, monkeypatch):
    from george_b200 import BasicSolver, _lib, kernels
    from george_b200._spec import flatten
    monkeypatch.delenv("BGP_BATCH_CHUNK", raising=False)
    lib = _lib.load()
    kernel = 1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3)
    spec = flatten(kernel)
    n = 1000
    params = _perturbed(kernel, 48, 13)
    x, sig, r = _inputs(n, 3, 48, 14)
    counts = []
    for nb in (1, 48):
        c0 = lib.bgp_launch_count()
        BasicSolver.batch_log_likelihood(spec, params[:nb], x, sig[:nb], r[:nb])
        counts.append(lib.bgp_launch_count() - c0)
    assert counts[0] == counts[1] > 0, counts


def test_hodlr_takes_the_loop_and_gp_pickles(gpu):
    import george_b200 as george
    from george_b200 import kernels
    rng = np.random.default_rng(15)
    x = np.sort(rng.uniform(0, 10, 400))
    y = np.sin(x) + 0.1 * rng.standard_normal(400)
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0), solver=george.HODLRSolver, tol=1e-12, min_size=50)
    gp.compute(x, 0.1)
    gp.log_likelihood(y)
    vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((4, len(gp)))
    st = _state(gp)
    got = gp.batch_log_likelihood(vecs, y)
    _assert_state(gp, st)
    assert np.array_equal(got, _loop(gp, vecs, y, False))

    gpd = george.GP(1.0 * kernels.ExpSquaredKernel(1.0))
    gpd.compute(x, 0.1)
    lld = gpd.log_likelihood(y)
    gpd.batch_log_likelihood(vecs, y)
    gp2 = pickle.loads(pickle.dumps(gpd))
    assert gp2.log_likelihood(y) == pytest.approx(lld, rel=1e-12, abs=1e-12)
    assert _close(gp2.batch_log_likelihood(vecs, y), gpd.batch_log_likelihood(vecs, y))


def test_large_batch(gpu):
    import george_b200 as george
    from george_b200 import kernels
    rng = np.random.default_rng(16)
    n = 4096
    x = rng.uniform(-3, 3, (n, 3))
    y = np.sin(x[:, 0]) * np.cos(x[:, 1]) + 0.1 * rng.standard_normal(n)
    gp = george.GP(1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3))
    gp.compute(x, 0.3)
    vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((32, len(gp)))
    got = gp.batch_log_likelihood(vecs, y)
    pick = [0, 9, 20, 31]
    assert np.all(np.isfinite(got))
    assert _close(got[pick], _loop(gp, vecs[pick], y, False))
