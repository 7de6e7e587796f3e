# -*- coding: utf-8 -*-
"""GP.batch_grad_predict / BasicSolver.batch_predict_grad on the device: every member's mean, variance and their
test-point gradients are the single path's (compute, apply_inverse, kernel.matvec, kernel.x1_gradient_matvec,
predictive_grad) bit for bit, mu and var are batch_predict's, failures stay with their member, the results do not
depend on B, the position or the chunking, the launch count does not grow with B, and the gradients are the central
differences of batch_predict."""
import pickle

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SIZES = [1, 63, 64, 65, 129, 300, 1000]
TEST_SIZES = [1, 8, 9, 65, 300]   # 8 | 9: either side of the few-column step kernels


def _zoo():
    from george_b200 import kernels as K
    return [
        ("expsq_1d", 1.0 * K.ExpSquaredKernel(1.0), 1),
        ("m32_1d", 2.3 * K.Matern32Kernel(0.7), 1),
        ("m52_1d", K.Matern52Kernel(0.9), 1),
        ("exp_1d", 0.7 * K.ExpKernel(1.1), 1),
        ("m52_3d_iso", K.Matern52Kernel(0.5, ndim=3), 3),
        ("m52_3d_axis", 1.3 * K.Matern52Kernel([0.5, 1.0, 2.0], ndim=3), 3),
        ("expsq_3d_general", K.ExpSquaredKernel([[1.0, 0.1, 0.2], [0.1, 2.0, 0.3], [0.2, 0.3, 1.5]], ndim=3), 3),
        ("sum_expsq_expsine2", 1.0 * K.ExpSquaredKernel(1.0, ndim=3)
         + 0.5 * K.ExpSine2Kernel(gamma=1.0, log_period=np.log(3.0), ndim=3, axes=1), 3),
        ("prod_m32_expsq", 0.9 * K.Matern32Kernel(1.5, ndim=2, axes=0) * K.ExpSquaredKernel(0.8, ndim=2, axes=1), 2),
        ("expsq_block", K.ExpSquaredKernel(1.0, ndim=3, block=[(-0.5, 0.5)] * 3), 3),
        ("user_cauchy", 0.8 * K.CauchyKernel(metric=0.7, ndim=2), 2),
        ("m32_4d_axis", K.Matern32Kernel([0.5, 1.0, 1.5, 2.0], ndim=4), 4),
        ("expsq_5d_iso", 1.1 * K.ExpSquaredKernel(2.0, ndim=5), 5),
        ("m52_6d_axis", K.Matern52Kernel([1.0, 1.5, 2.0, 2.5, 3.0, 3.5], ndim=6), 6),
        ("ratquad_7d", K.RationalQuadraticKernel(log_alpha=0.3, metric=3.0, ndim=7), 7),
        ("expsq_8d_axis", 0.6 * K.ExpSquaredKernel(np.linspace(1.0, 4.0, 8), ndim=8), 8),
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


def _single(kernel, p, x, sig, r, xs):
    """GP.grad_predict's device steps for one member: compute, apply_inverse (alpha), kernel.matvec,
    kernel.x1_gradient_matvec and predictive_grad.  Returns (mean, var, dmu, dvar)."""
    from george_b200 import BasicSolver
    p0 = kernel.get_parameter_vector(include_frozen=True)
    kernel.set_parameter_vector(p, include_frozen=True)
    try:
        s = BasicSolver(kernel)
        s.compute(x, sig)
        alpha = s.apply_inverse(np.array(r), in_place=True).flatten()
        mean = kernel.matvec(xs, x, alpha)
        dmu = kernel.kernel.x1_gradient_matvec(xs, x, alpha)
        var, dvar = s.predictive_grad(kernel, xs)
        return mean, var, dmu, dvar
    finally:
        kernel.set_parameter_vector(p0, include_frozen=True)


def _check_members(kernel, params, x, sig, r, xs):
    from george_b200 import BasicSolver
    from george_b200._spec import flatten
    spec = flatten(kernel)
    singles = [_single(kernel, params[b], x, sig[b], r[b], xs) for b in range(len(params))]
    for rv in (False, True):
        mean, var, dmu, dvar, info = BasicSolver.batch_predict_grad(spec, params, x, sig, r, xs, rv)
        assert np.all(info == 0), (rv, info)
        assert dmu.shape == (len(params), len(xs), x.shape[1])
        if not rv:
            assert var is None and dvar is None
        for b, (m1, v1, dm1, dv1) in enumerate(singles):
            assert np.array_equal(mean[b], m1), (rv, b)
            assert np.array_equal(dmu[b], dm1), (rv, b, np.max(np.abs(dmu[b] - dm1)))
            if rv:
                assert np.array_equal(var[b], v1), (b, np.max(np.abs(var[b] - v1)))
                assert np.array_equal(dvar[b], dv1), (b, np.max(np.abs(dvar[b] - dv1)))


@pytest.mark.parametrize("name", [z[0] for z in _zoo()])
def test_members_match_the_single_path(gpu, name):
    _, kernel, ndim = [z for z in _zoo() if z[0] == name][0]
    for n in SIZES:
        for ns in TEST_SIZES:
            params = _perturbed(kernel, 2, 100 * n + ns)
            x, xs, sig, r = _inputs(n, ns, ndim, 2, n + ns)
            _check_members(kernel, params, x, sig, r, xs)


@pytest.mark.parametrize("chunk", ["1", "8", "9", "64"])
def test_ragged_test_point_chunks(gpu, monkeypatch, chunk):
    """Forced test-point chunk widths that leave a ragged tail: every chunk, on either side of the step kernels."""
    from george_b200 import kernels
    monkeypatch.setenv("BGP_PREDICT_CHUNK", chunk)
    for kernel, ndim in ((1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3), 3),
                         (2.3 * kernels.Matern32Kernel(0.7), 1),
                         (0.8 * kernels.CauchyKernel(metric=0.7, ndim=2), 2)):
        for n in (65, 300):
            params = _perturbed(kernel, 3, n)
            x, xs, sig, r = _inputs(n, 67, ndim, 3, n + 1)
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


def _matern_gp(n=500, seed=1):
    import george_b200 as george
    from george_b200 import kernels
    rng = np.random.default_rng(seed)
    x = rng.uniform(-3, 3, (n, 3))
    y = 0.4 + np.sin(x[:, 0]) * np.cos(x[:, 1]) + 0.1 * rng.standard_normal(n)
    gp = george.GP(1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3), mean=0.4, fit_mean=True,
                   white_noise=np.log(0.05), fit_white_noise=True)
    gp.compute(x, 0.2)
    return gp, y


def _state(gp):
    return (gp.get_parameter_vector(include_frozen=True).copy(), gp.computed, gp.solver, gp._alpha, gp._y,
            gp._const, [m.dirty for m in gp.models.values()])


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
            res.append(gp.grad_predict(y, t, **kw))
    finally:
        gp.set_parameter_vector(p0)
    return tuple(np.stack([q[k] for q in res]) for k in range(len(res[0])))


def _equal(got, want):
    return len(got) == len(want) and all(a.shape == b.shape and np.array_equal(a, b) for a, b in zip(got, want))


def _check_gp(gp, y, vecs, t):
    gp.log_likelihood(y)
    ref = gp.grad_predict(y, t, return_var=True)
    for rv in (False, True):
        st = _state(gp)
        got = gp.batch_grad_predict(vecs, y, t, return_var=rv)
        _assert_state(gp, st)
        assert _equal(gp.grad_predict(y, t, return_var=True), ref)  # the same factorisation and cached solve
        assert gp._alpha is st[3]
        want = _loop(gp, vecs, y, t, return_var=rv)
        assert _equal(got, want), rv
        # mu and var are batch_predict's
        bp = gp.batch_predict(vecs, y, t, return_var=True)
        assert np.array_equal(got[0], bp[0])
        if rv:
            assert np.array_equal(got[1], bp[1])
        gp.log_likelihood(y)  # (the reference loop above left the GP at another factorisation)
        ref = gp.grad_predict(y, t, return_var=True)


def test_co2_posterior(gpu):
    gp, y = _co2_gp()
    rng = np.random.default_rng(5)
    vecs = gp.get_parameter_vector() + 1e-4 * rng.standard_normal((6, len(gp)))
    _check_gp(gp, y, vecs, np.linspace(1950, 2010, 120))
    _check_gp(gp, y, vecs, np.array([1990.5]))


def test_fitted_constant_mean_and_white_noise(gpu):
    gp, y = _matern_gp()
    rng = np.random.default_rng(6)
    vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((5, len(gp)))
    _check_gp(gp, y, vecs, rng.uniform(-3, 3, (70, 3)))
    gp.freeze_parameter("white_noise:value")
    vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((4, len(gp)))
    _check_gp(gp, y, vecs, rng.uniform(-3, 3, (9, 3)))


def test_results_do_not_depend_on_batch_position_or_chunking(gpu, monkeypatch):
    from george_b200 import BasicSolver, kernels
    from george_b200._spec import flatten
    kernel = 1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3)
    spec = flatten(kernel)
    n, ns, nb = 130, 70, 12
    params = _perturbed(kernel, nb, 11)
    x, xs, sig, r = _inputs(n, ns, 3, nb, 12)
    monkeypatch.delenv("BGP_BATCH_CHUNK", raising=False)

    def run(idx, rv):
        return BasicSolver.batch_predict_grad(spec, params[idx], x, sig[idx], r[idx], xs, rv)[:4]

    def same(a, b, ia, ib):
        return all((p is None and q is None) or np.array_equal(p[ia], q[ib]) for p, q in zip(a, b))

    for rv in (False, True):
        full = run(slice(None), rv)
        assert same(full, run(slice(None), rv), slice(None), slice(None))
        for b in (0, 5, 11):
            assert same(run(slice(b, b + 1), rv), full, 0, b), (rv, b)
        order = [i for i in range(nb) if i != 5] + [5]
        assert same(run(order, rv), full, -1, 5)
        for chunk in ("1", "5", str(nb)):
            monkeypatch.setenv("BGP_BATCH_CHUNK", chunk)
            got = run(slice(None), rv)
            monkeypatch.delenv("BGP_BATCH_CHUNK")
            assert same(got, full, slice(None), slice(None)), (rv, chunk)


@pytest.mark.parametrize("return_var", [False, True])
def test_launch_count_does_not_grow_with_the_batch(gpu, monkeypatch, return_var):
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
        BasicSolver.batch_predict_grad(spec, params[:nb], x, sig[:nb], r[:nb], xs, return_var)
        counts.append(lib.bgp_launch_count() - c0)
    assert counts[0] == counts[1] > 0, counts


def _dot_gp():
    import george_b200 as george
    from george_b200 import kernels
    x = np.linspace(0.1, 1, 50)
    gp = george.GP(kernels.DotProductKernel(), mean=0.1, fit_mean=True, white_noise=np.log(0.1),
                   fit_white_noise=True)
    gp.compute(x, 0.0)
    y = np.cos(x)
    return gp, y


def test_failures_stay_with_their_member(gpu):
    from george_b200 import BasicSolver
    from george_b200._spec import flatten
    gp, y = _dot_gp()
    t = np.linspace(0, 1.2, 20)
    vecs = np.tile(gp.get_parameter_vector(), (8, 1))
    bad = [2, 5]
    vecs[bad, 1] = -80.0  # K = x x^T + 1.8e-35 I: rank one, not positive definite
    gp.log_likelihood(y)
    for rv in (False, True):
        st = _state(gp)
        with pytest.raises(np.linalg.LinAlgError) as batch_exc:
            gp.batch_grad_predict(vecs, y, t, return_var=rv)
        _assert_state(gp, st)
        with pytest.raises(np.linalg.LinAlgError) as loop_exc:
            _loop(gp, vecs, y, t, return_var=rv)
        assert str(batch_exc.value) == str(loop_exc.value)
        gp.log_likelihood(y)

    # a non-finite constant mean: the loop's ValueError, raised for the first failing member (here before member 5's
    # factorisation error)
    v2 = vecs.copy()
    v2[1, 0] = np.nan
    st = _state(gp)
    with pytest.raises(ValueError) as batch_exc:
        gp.batch_grad_predict(v2, y, t, return_var=True)
    _assert_state(gp, st)
    with pytest.raises(ValueError) as loop_exc:
        _loop(gp, v2, y, t, return_var=True)
    assert "mean function" in str(batch_exc.value) and str(batch_exc.value) == str(loop_exc.value)
    gp.log_likelihood(y)

    # through the ABI: the good members are the single path's, the bad ones NaN with the single path's minor index
    x = gp._x
    sig = np.sqrt(np.zeros((8, 50)) + np.exp(vecs[:, 1:2]))
    r = np.tile(y - 0.1, (8, 1))
    xs = t[:, None]
    mean, var, dmu, dvar, info = BasicSolver.batch_predict_grad(flatten(gp.kernel), np.zeros((8, 0)), x, sig, r, xs,
                                                                True)
    for b in range(8):
        if b in bad:
            with pytest.raises(np.linalg.LinAlgError) as e:
                BasicSolver(gp.kernel).compute(x, sig[b])
            assert info[b] > 0 and str(e.value).startswith("%d-th" % info[b])
            assert all(np.all(np.isnan(a[b])) for a in (mean, var, dmu, dvar))
        else:
            assert info[b] == 0
            want = _single(gp.kernel, np.zeros(0), x, sig[b], r[b], xs)
            assert all(np.array_equal(a[b], w) for a, w in zip((mean, var, dmu, dvar), want))


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
    for rv in (False, True):
        st = _state(gp)
        got = gp.batch_grad_predict(vecs, y, t, return_var=rv)
        _assert_state(gp, st)
        assert _equal(got, _loop(gp, vecs, y, t, return_var=rv))
        gp.log_likelihood(y)

    gpd = george.GP(1.0 * kernels.ExpSquaredKernel(1.0))
    gpd.compute(x, 0.1)
    gpd.log_likelihood(y)
    k2 = 0.5 * kernels.Matern32Kernel(2.0)
    for rv in (False, True):
        st = _state(gpd)
        got = gpd.batch_grad_predict(vecs, y, t, return_var=rv, kernel=k2)
        _assert_state(gpd, st)
        assert _equal(got, _loop(gpd, vecs, y, t, return_var=rv, kernel=k2))
        gpd.log_likelihood(y)
    want = gpd.batch_grad_predict(vecs, y, t, return_var=True)
    gp2 = pickle.loads(pickle.dumps(gpd))
    assert _equal(gp2.batch_grad_predict(vecs, y, t, return_var=True), want)
    assert _equal(want, _loop(gpd, vecs, y, t, return_var=True))


def test_large_batch(gpu, monkeypatch):
    """B = 256 at n = 1000 over member chunks of 100 (two full chunks and a ragged one)."""
    import george_b200 as george
    from george_b200 import kernels
    rng = np.random.default_rng(16)
    n = 1000
    x = rng.uniform(-3, 3, (n, 3))
    y = np.sin(x[:, 0]) * np.cos(x[:, 1]) + 0.1 * rng.standard_normal(n)
    t = rng.uniform(-3, 3, (64, 3))
    gp = george.GP(1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3))
    gp.compute(x, 0.3)
    vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((256, len(gp)))
    monkeypatch.setenv("BGP_BATCH_CHUNK", "100")
    got = gp.batch_grad_predict(vecs, y, t, return_var=True)
    monkeypatch.delenv("BGP_BATCH_CHUNK")
    assert all(np.all(np.isfinite(a)) for a in got)
    pick = [0, 99, 100, 199, 200, 255]
    assert _equal(tuple(a[pick] for a in got), _loop(gp, vecs[pick], y, t, return_var=True))
    assert _equal(got, gp.batch_grad_predict(vecs, y, t, return_var=True))


def test_gradients_are_central_differences_of_batch_predict(gpu):
    """dmu and dvar against (f(t + h e_q) - f(t - h e_q)) / 2h of batch_predict, independently of the loop."""
    gp, y = _matern_gp(n=300, seed=3)
    rng = np.random.default_rng(17)
    vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((4, len(gp)))
    t = rng.uniform(-2.5, 2.5, (25, 3))
    mu, var, dmu, dvar = gp.batch_grad_predict(vecs, y, t, return_var=True)
    h = 1e-5
    for q in range(3):
        e = np.zeros(3)
        e[q] = h
        mp, vp = gp.batch_predict(vecs, y, t + e, return_var=True)
        mm, vm = gp.batch_predict(vecs, y, t - e, return_var=True)
        fd_mu, fd_var = (mp - mm) / (2 * h), (vp - vm) / (2 * h)
        assert np.allclose(dmu[:, :, q], fd_mu, rtol=1e-5, atol=1e-6 * np.max(np.abs(fd_mu))), q
        assert np.allclose(dvar[:, :, q], fd_var, rtol=1e-4, atol=1e-5 * np.max(np.abs(fd_var))), q
