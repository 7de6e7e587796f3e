# -*- coding: utf-8 -*-
"""GP.batch_predict / BasicSolver.batch_predict on the device: every member's mean, variance and covariance are the
single path's (compute, apply_inverse, kernel.matvec, predictive) bit for bit, failures stay with their member, the
results do not depend on B, the position or the chunking, and the launch count does not grow with B."""
import pickle

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SIZES = [1, 2, 63, 64, 65, 129, 300, 1000]
TEST_SIZES = [1, 8, 9, 65, 300]   # 8 | 9: either side of the few-column step kernels
WHATS = [None, "var", "cov"]


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


def _inputs(n, ns, ndim, nb, seed):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-2, 2, (n, ndim))
    xs = rng.uniform(-2.5, 2.5, (ns, ndim))
    sig = 0.5 + 0.5 * rng.uniform(size=(nb, n))
    r = rng.standard_normal((nb, n))
    return x, xs, sig, r


def _perturbed(kernel, nb, seed, scale=0.05):
    rng = np.random.default_rng(seed)
    p0 = kernel.get_parameter_vector(include_frozen=True)
    return p0 + scale * rng.standard_normal((nb, len(p0)))


def _single(kernel, p, x, sig, r, xs, what):
    """GP.predict's device steps for one member: compute, apply_inverse (alpha), kernel.matvec, predictive."""
    from george_b200 import BasicSolver
    p0 = kernel.get_parameter_vector(include_frozen=True)
    kernel.set_parameter_vector(p, include_frozen=True)
    try:
        s = BasicSolver(kernel)
        s.compute(x, sig)
        alpha = s.apply_inverse(np.array(r), in_place=True).flatten()
        mean = kernel.matvec(xs, x, alpha)
        return mean, (s.predictive(kernel, xs, what) if what else None)
    finally:
        kernel.set_parameter_vector(p0, include_frozen=True)


def _check_members(kernel, params, x, sig, r, xs, members=None):
    from george_b200 import BasicSolver
    from george_b200._spec import flatten
    for what in WHATS:
        mean, out, info = BasicSolver.batch_predict(flatten(kernel), params, x, sig, r, xs, what)
        assert np.all(info == 0), (what, info)
        for b in (range(len(params)) if members is None else members):
            m1, o1 = _single(kernel, params[b], x, sig[b], r[b], xs, what)
            assert np.array_equal(mean[b], m1), (what, b, np.max(np.abs(mean[b] - m1)))
            if what is None:
                assert out is None
            else:
                assert np.array_equal(out[b], o1), (what, b, np.max(np.abs(out[b] - o1)))


@pytest.mark.parametrize("name", [z[0] for z in _zoo()])
def test_members_match_the_single_path(gpu, name):
    _, kernel, ndim = [z for z in _zoo() if z[0] == name][0]
    for n in SIZES:
        for ns in TEST_SIZES:
            params = _perturbed(kernel, 2, 100 * n + ns)
            x, xs, sig, r = _inputs(n, ns, ndim, 2, n + ns)
            _check_members(kernel, params, x, sig, r, xs)


def test_ragged_test_point_chunks(gpu, monkeypatch):
    from george_b200 import kernels
    monkeypatch.setenv("BGP_PREDICT_CHUNK", "64")
    for kernel, ndim in ((1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3), 3),
                         (0.8 * kernels.CauchyKernel(metric=0.7, ndim=2), 2)):
        for n in (65, 300):
            params = _perturbed(kernel, 3, n)
            x, xs, sig, r = _inputs(n, 300, ndim, 3, n + 1)
            _check_members(kernel, params, x, sig, r, xs)


def _co2_gp(n=300, seed=0):
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
            gp.kernel.dirty, gp._const)


def _assert_state(gp, st):
    now = _state(gp)
    assert np.array_equal(st[0], now[0])
    assert now[1] == st[1] and now[5] == st[5] and now[6] == st[6]
    assert now[2] is st[2] and now[3] is st[3] and now[4] is st[4]


def _loop(gp, vecs, y, t, **kw):
    p0 = gp.get_parameter_vector()
    res = []
    try:
        for v in vecs:
            gp.set_parameter_vector(v)
            res.append(gp.predict(y, t, **kw))
    finally:
        gp.set_parameter_vector(p0)
    if isinstance(res[0], tuple):
        return np.stack([q[0] for q in res]), np.stack([q[1] for q in res])
    return np.stack(res)


def _equal(got, want):
    if isinstance(want, tuple):
        return isinstance(got, tuple) and all(np.array_equal(a, b) for a, b in zip(got, want))
    return np.array_equal(got, want)


def _check_gp(gp, y, vecs, t):
    gp.log_likelihood(y)
    ref = gp.predict(y, t, return_var=True)
    for kw in (dict(return_cov=False), dict(return_var=True), dict()):
        st = _state(gp)
        got = gp.batch_predict(vecs, y, t, **kw)
        _assert_state(gp, st)
        assert gp.solver is st[2]
        assert _equal(gp.predict(y, t, return_var=True), ref)  # the same factorisation and cached solve
        assert gp._alpha is st[3]
        want = _loop(gp, vecs, y, t, **kw)
        assert _equal(got, want), kw
        gp.log_likelihood(y)  # (the reference loop above left the GP at another factorisation)
        ref = gp.predict(y, t, return_var=True)


def test_co2_posterior_predictive(gpu):
    gp, y = _co2_gp()
    rng = np.random.default_rng(5)
    vecs = gp.get_parameter_vector() + 1e-4 * rng.standard_normal((6, len(gp)))
    _check_gp(gp, y, vecs, np.linspace(1950, 2010, 120))


def test_non_constant_mean_with_frozen_parameters(gpu):
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
    vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((5, len(gp)))
    _check_gp(gp, y, vecs, np.linspace(-6, 6, 70))
    assert np.array_equal(gp.mean.get_parameter_vector(include_frozen=True), [0.4, 0.0])


def test_results_do_not_depend_on_batch_position_or_chunking(gpu, monkeypatch):
    from george_b200 import BasicSolver, kernels
    from george_b200._spec import flatten
    kernel = 1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3)
    spec = flatten(kernel)
    n, ns, nb = 130, 70, 12
    params = _perturbed(kernel, nb, 11)
    x, xs, sig, r = _inputs(n, ns, 3, nb, 12)
    monkeypatch.delenv("BGP_BATCH_CHUNK", raising=False)
    for what in WHATS:
        mu, out, _ = BasicSolver.batch_predict(spec, params, x, sig, r, xs, what)
        mu2, out2, _ = BasicSolver.batch_predict(spec, params, x, sig, r, xs, what)
        assert np.array_equal(mu, mu2) and (what is None or np.array_equal(out, out2))
        for b in (0, 5, 11):
            m1, o1, _ = BasicSolver.batch_predict(spec, params[b:b + 1], x, sig[b:b + 1], r[b:b + 1], xs, what)
            assert np.array_equal(m1[0], mu[b]) and (what is None or np.array_equal(o1[0], out[b])), (what, b)
        order = [i for i in range(nb) if i != 5] + [5]
        m3, o3, _ = BasicSolver.batch_predict(spec, params[order], x, sig[order], r[order], xs, what)
        assert np.array_equal(m3[-1], mu[5]) and (what is None or np.array_equal(o3[-1], out[5]))
        for chunk in ("1", "5", str(nb)):
            monkeypatch.setenv("BGP_BATCH_CHUNK", chunk)
            mc, oc, _ = BasicSolver.batch_predict(spec, params, x, sig, r, xs, what)
            monkeypatch.delenv("BGP_BATCH_CHUNK")
            assert np.array_equal(mc, mu) and (what is None or np.array_equal(oc, out)), (what, chunk)


@pytest.mark.parametrize("what", ["var", "cov"])
def test_launch_count_does_not_grow_with_the_batch(gpu, monkeypatch, what):
    from george_b200 import BasicSolver, _lib, kernels
    from george_b200._spec import flatten
    monkeypatch.delenv("BGP_BATCH_CHUNK", raising=False)
    lib = _lib.load()
    kernel = 1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3)
    spec = flatten(kernel)
    n, ns = 1000, 100
    params = _perturbed(kernel, 48, 13)
    x, xs, sig, r = _inputs(n, ns, 3, 48, 14)
    counts = []
    for nb in (1, 48):
        c0 = lib.bgp_launch_count()
        BasicSolver.batch_predict(spec, params[:nb], x, sig[:nb], r[:nb], xs, what)
        counts.append(lib.bgp_launch_count() - c0)
    assert counts[0] == counts[1] > 0, counts


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
    from george_b200._spec import flatten
    gp, y = _dot_gp()
    t = np.linspace(0, 1.2, 20)
    vecs = np.full((8, len(gp)), np.log(0.1))
    bad = [2, 5]
    vecs[bad, 0] = -80.0  # K = x x^T + 1.8e-35 I: rank one, not positive definite
    gp.log_likelihood(y)
    st = _state(gp)
    with pytest.raises(np.linalg.LinAlgError) as batch_exc:
        gp.batch_predict(vecs, y, t, return_var=True)
    _assert_state(gp, st)
    with pytest.raises(np.linalg.LinAlgError) as loop_exc:
        _loop(gp, vecs, y, t, return_var=True)
    assert str(batch_exc.value) == str(loop_exc.value)

    # through the ABI: the good members are the single path's, the bad ones NaN with the single path's minor index
    x = gp._x
    sig = np.sqrt(np.zeros((8, 50)) + np.exp(vecs[:, :1]))
    r = np.tile(y, (8, 1))
    xs = t[:, None]
    for what in WHATS:
        mean, out, info = BasicSolver.batch_predict(flatten(gp.kernel), np.zeros((8, 0)), x, sig, r, xs, what)
        for b in range(8):
            if b in bad:
                with pytest.raises(np.linalg.LinAlgError) as e:
                    BasicSolver(gp.kernel).compute(x, sig[b])
                assert info[b] > 0 and str(e.value).startswith("%d-th" % info[b])
                assert np.all(np.isnan(mean[b])) and (what is None or np.all(np.isnan(out[b])))
            else:
                assert info[b] == 0
                m1, o1 = _single(gp.kernel, np.zeros(0), x, sig[b], r[b], xs, what)
                assert np.array_equal(mean[b], m1) and (what is None or np.array_equal(out[b], o1))


def test_hodlr_and_explicit_kernel_take_the_loop_and_gp_pickles(gpu):
    import george_b200 as george
    from george_b200 import kernels
    rng = np.random.default_rng(15)
    x = np.sort(rng.uniform(0, 10, 400))
    y = np.sin(x) + 0.1 * rng.standard_normal(400)
    t = np.linspace(-1, 11, 50)
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0), solver=george.HODLRSolver, tol=1e-12, min_size=50)
    gp.compute(x, 0.1)
    gp.log_likelihood(y)
    vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((3, len(gp)))
    for kw in (dict(return_cov=False), dict(return_var=True)):
        st = _state(gp)
        got = gp.batch_predict(vecs, y, t, **kw)
        _assert_state(gp, st)
        assert _equal(got, _loop(gp, vecs, y, t, **kw))
        gp.log_likelihood(y)

    gpd = george.GP(1.0 * kernels.ExpSquaredKernel(1.0))
    gpd.compute(x, 0.1)
    gpd.log_likelihood(y)
    k2 = 0.5 * kernels.Matern32Kernel(2.0)
    for kw in (dict(return_cov=False), dict(return_var=True), dict()):
        got = gpd.batch_predict(vecs, y, t, kernel=k2, **kw)
        assert _equal(got, _loop(gpd, vecs, y, t, kernel=k2, **kw))
    gpd.log_likelihood(y)
    want = gpd.batch_predict(vecs, y, t, return_var=True)
    gp2 = pickle.loads(pickle.dumps(gpd))
    assert _equal(gp2.batch_predict(vecs, y, t, return_var=True), want)
    assert _equal(want, _loop(gpd, vecs, y, t, return_var=True))


def test_large_batch(gpu):
    import george_b200 as george
    from george_b200 import kernels
    rng = np.random.default_rng(16)
    n = 4096
    x = rng.uniform(-3, 3, (n, 3))
    y = np.sin(x[:, 0]) * np.cos(x[:, 1]) + 0.1 * rng.standard_normal(n)
    t = rng.uniform(-3, 3, (500, 3))
    gp = george.GP(1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3))
    gp.compute(x, 0.3)
    vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((32, len(gp)))
    mu, var = gp.batch_predict(vecs, y, t, return_var=True)
    pick = [0, 9, 20, 31]
    assert np.all(np.isfinite(mu)) and np.all(np.isfinite(var))
    assert _equal((mu[pick], var[pick]), _loop(gp, vecs[pick], y, t, return_var=True))
