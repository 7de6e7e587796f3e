# -*- coding: utf-8 -*-
"""GP.batch_sample_conditional / BasicSolver.batch_sample on the device: every member's draws are the single path's
(compute, apply_inverse, kernel.matvec + the mean model, sample_predictive) bit for bit, the GP result is the
per-vector loop's, failures stay with their member, the results do not depend on B, the position or the chunking, and
the launch count does not grow with B."""
import pickle
import re

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SIZES = [1, 63, 64, 65, 300]
TEST_SIZES = [1, 8, 9, 65, 300]
DRAWS = [1, 7, 8, 129]   # 7 | 8: either side of BGP_SAMPLE_DMMA_ROWS
JITTER = 1e-6


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


def _single(kernel, p, x, sig, r, xs, mean_add, z, jitter):
    """GP.sample_conditional's device steps for one member: the draws, or the LinAlgError the covariance raises."""
    from george_b200 import BasicSolver
    p0 = kernel.get_parameter_vector(include_frozen=True)
    kernel.set_parameter_vector(p, include_frozen=True)
    try:
        s = BasicSolver(kernel)
        s.compute(x, sig)
        alpha = s.apply_inverse(np.array(r), in_place=True).flatten()
        mean = kernel.matvec(xs, x, alpha) + mean_add
        try:
            return s.sample_predictive(kernel, xs, mean, z, jitter)
        except np.linalg.LinAlgError as e:
            return e
    finally:
        kernel.set_parameter_vector(p0, include_frozen=True)


def _minor(exc):
    return int(re.match(r"(\d+)-th leading minor", str(exc)).group(1))


def _check_members(kernel, params, x, sig, r, xs, size, jitter=JITTER, seed=0):
    """Every member against the single path; returns the number of members that drew."""
    from george_b200 import BasicSolver
    from george_b200._spec import flatten
    nb, ns = len(params), len(xs)
    rng = np.random.default_rng(seed)
    mean_add = rng.standard_normal((nb, ns))
    z = rng.standard_normal((nb, size, ns))
    draws, info, draw_info = BasicSolver.batch_sample(flatten(kernel), params, x, sig, r, xs, mean_add, z, jitter)
    assert np.all(info == 0), info
    drew = 0
    for b in range(nb):
        want = _single(kernel, params[b], x, sig[b], r[b], xs, mean_add[b], z[b], jitter)
        if isinstance(want, Exception):
            assert draw_info[b] == _minor(want), (b, draw_info[b], str(want))
            assert np.all(np.isnan(draws[b]))
        else:
            assert draw_info[b] == 0, (b, draw_info[b])
            assert np.array_equal(draws[b], want), (b, np.max(np.abs(draws[b] - want)))
            drew += 1
    return drew


@pytest.mark.parametrize("name", [z[0] for z in _zoo()])
def test_members_match_the_single_path(gpu, name):
    _, kernel, ndim = [z for z in _zoo() if z[0] == name][0]
    drew = 0
    for n in SIZES:
        for ns in TEST_SIZES:
            params = _perturbed(kernel, 2, 100 * n + ns)
            x, xs, sig, r = _inputs(n, ns, ndim, 2, n + ns)
            for size in DRAWS:
                drew += _check_members(kernel, params, x, sig, r, xs, size, seed=size)
    assert drew > 0


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


def _gen_state(rng):
    return rng.bit_generator.state if isinstance(rng, np.random.Generator) else rng.get_state()


def _same_gen(a, b):
    sa, sb = _gen_state(a), _gen_state(b)
    if isinstance(sa, dict):
        return sa == sb
    return sa[0] == sb[0] and np.array_equal(sa[1], sb[1]) and sa[2:] == sb[2:]


def _loop(gp, vecs, y, t, size, **kw):
    p0 = gp.get_parameter_vector()
    try:
        res = []
        for v in vecs:
            gp.set_parameter_vector(v)
            res.append(gp.sample_conditional(y, t, size, **kw))
    finally:
        gp.set_parameter_vector(p0)
    return np.stack(res)


def _check_gp(gp, y, vecs, t, jitter=None):
    """batch vs loop for both generator types and several sizes; returns the number of comparisons that drew."""
    drew = 0
    for make in (np.random.default_rng, np.random.RandomState):
        for size in (1, 5, 8, 40):
            gp.log_likelihood(y)
            st = _state(gp)
            g1, g2 = make(size), make(size)
            try:
                got = gp.batch_sample_conditional(vecs, y, t, size, rng=g1, jitter=jitter)
            except np.linalg.LinAlgError as e:
                got = e
            _assert_state(gp, st)
            try:
                want = _loop(gp, vecs, y, t, size, rng=g2, jitter=jitter)
            except np.linalg.LinAlgError as e:
                want = e
            if isinstance(want, Exception):
                assert isinstance(got, type(want)) and str(got) == str(want)
                continue
            assert not isinstance(got, Exception), str(got)
            assert got.shape == want.shape and np.array_equal(got, want), (make, size)
            assert _same_gen(g1, g2)
            drew += 1
    return drew


def test_co2_posterior_draws(gpu):
    gp, y = _co2_gp()
    rng = np.random.default_rng(5)
    vecs = gp.get_parameter_vector() + 1e-4 * rng.standard_normal((6, len(gp)))
    t = np.linspace(1950, 2010, 60)
    assert _check_gp(gp, y, vecs, t, jitter=1e-4) == 8
    _check_gp(gp, y, vecs, t)  # the default jitter: the same draws, or the same error


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
    assert _check_gp(gp, y, vecs, np.linspace(-6, 6, 70), jitter=1e-6) == 8
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
    for size in (1, 16):
        g = np.random.default_rng(size)
        madd, z = g.standard_normal((nb, ns)), g.standard_normal((nb, size, ns))

        def run(idx):
            return BasicSolver.batch_sample(spec, params[idx], x, sig[idx], r[idx], xs, madd[idx], z[idx], JITTER)[0]

        full = run(slice(None))
        assert np.all(np.isfinite(full))
        assert np.array_equal(full, run(slice(None)))
        for b in (0, 5, 11):
            assert np.array_equal(run(slice(b, b + 1))[0], full[b]), (size, b)
        order = [i for i in range(nb) if i != 5] + [5]
        assert np.array_equal(run(order)[-1], full[5])
        for chunk in ("1", "5", str(nb)):
            monkeypatch.setenv("BGP_BATCH_CHUNK", chunk)
            got = run(slice(None))
            monkeypatch.delenv("BGP_BATCH_CHUNK")
            assert np.array_equal(got, full), (size, chunk)


@pytest.mark.parametrize("size", [1, 16])
def test_launch_count_does_not_grow_with_the_batch(gpu, monkeypatch, size):
    from george_b200 import BasicSolver, _lib, kernels
    from george_b200._spec import flatten
    monkeypatch.delenv("BGP_BATCH_CHUNK", raising=False)
    lib = _lib.load()
    kernel = 1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3)
    spec = flatten(kernel)
    n, ns = 1000, 100
    params = _perturbed(kernel, 48, 13)
    x, xs, sig, r = _inputs(n, ns, 3, 48, 14)
    g = np.random.default_rng(0)
    madd, z = g.standard_normal((48, ns)), g.standard_normal((48, size, ns))
    counts = []
    for nb in (1, 48):
        c0 = lib.bgp_launch_count()
        BasicSolver.batch_sample(spec, params[:nb], x, sig[:nb], r[:nb], xs, madd[:nb], z[:nb], JITTER)
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


def test_a_member_whose_k_is_not_positive_definite_raises_the_loops_error(gpu):
    gp, y = _dot_gp()
    t = np.linspace(0, 1.2, 20)
    vecs = np.full((8, len(gp)), np.log(0.1))
    vecs[[2, 5], 0] = -80.0  # K = x x^T + 1.8e-35 I: rank one, not positive definite
    gp.log_likelihood(y)
    st = _state(gp)
    with pytest.raises(np.linalg.LinAlgError) as batch_exc:
        gp.batch_sample_conditional(vecs, y, t, 3, rng=np.random.default_rng(0), jitter=1e-6)
    _assert_state(gp, st)
    with pytest.raises(np.linalg.LinAlgError) as loop_exc:
        _loop(gp, vecs, y, t, 3, rng=np.random.default_rng(0), jitter=1e-6)
    assert str(batch_exc.value) == str(loop_exc.value)


def test_a_singular_predictive_covariance_raises_the_loops_error(gpu):
    import george_b200 as george
    from george_b200 import kernels
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0))
    gp.compute(np.linspace(0, 3, 10), 1e-3)
    y = np.zeros(10)
    ts = np.array([5.0, 5.0, 6.0])
    vecs = gp.get_parameter_vector() + np.array([[0.0], [0.1], [0.2]])
    gp.log_likelihood(y)
    st = _state(gp)
    with pytest.raises(np.linalg.LinAlgError, match="2-th leading minor.*larger jitter") as batch_exc:
        gp.batch_sample_conditional(vecs, y, ts, rng=np.random.default_rng(0), jitter=0.0)
    _assert_state(gp, st)
    with pytest.raises(np.linalg.LinAlgError) as loop_exc:
        _loop(gp, vecs, y, ts, 1, rng=np.random.default_rng(0), jitter=0.0)
    assert str(batch_exc.value) == str(loop_exc.value)
    got = gp.batch_sample_conditional(vecs, y, ts, rng=np.random.default_rng(0), jitter=1e-6)
    assert np.array_equal(got, _loop(gp, vecs, y, ts, 1, rng=np.random.default_rng(0), jitter=1e-6))


def test_failures_stay_with_their_member(gpu):
    """Through the ABI: members that fail the K factorisation (info) and members that fail only the covariance
    Cholesky (draw_info), each outcome taken from the single path."""
    from george_b200 import BasicSolver, kernels
    from george_b200._spec import flatten
    gp, y = _dot_gp()
    x = gp._x
    t = np.linspace(0, 1.2, 20)
    sig2 = np.full((8, 50), np.exp(np.log(0.1)))
    sig2[[2, 5]] = np.exp(-80.0)
    sig = np.sqrt(sig2)
    r = np.tile(y, (8, 1))
    g = np.random.default_rng(1)
    madd, z = g.standard_normal((8, 20)), g.standard_normal((8, 3, 20))
    draws, info, draw_info = BasicSolver.batch_sample(flatten(gp.kernel), np.zeros((8, 0)), x, sig, r, t[:, None],
                                                      madd, z, 1e-6)
    for b in range(8):
        if b in (2, 5):
            with pytest.raises(np.linalg.LinAlgError) as e:
                BasicSolver(gp.kernel).compute(x, sig[b])
            assert info[b] == _minor(e.value) and draw_info[b] == 0
            assert np.all(np.isnan(draws[b]))
        else:
            assert info[b] == 0
            want = _single(gp.kernel, np.zeros(0), x, sig[b], r[b], t[:, None], madd[b], z[b], 1e-6)
            assert np.array_equal(draws[b], want)

    # near-duplicate test points with jitter 0: the covariance loses positive definiteness for the longer length
    # scales only; with two members that cannot factorise K in between
    kernel = 1.0 * kernels.ExpSquaredKernel(1.0)
    rng = np.random.default_rng(2)
    xk = np.sort(rng.uniform(0, 3, 40))[:, None]
    xs = np.array([4.0, 4.0 + 1e-7, 4.5, 5.0])[:, None]
    nb = 10
    params = np.tile(kernel.get_parameter_vector(include_frozen=True), (nb, 1))
    params[:, 1] = np.linspace(np.log(0.05), np.log(20.0), nb)  # the metric: length scales from short to long
    sigk = np.full((nb, 40), 0.1)
    sigk[[3, 8]] = 0.0
    params[[3, 8], 1] = np.log(50.0)  # a smooth kernel without noise: K itself is not positive definite
    rk = np.tile(np.sin(xk[:, 0]), (nb, 1))
    madd, z = rng.standard_normal((nb, 4)), rng.standard_normal((nb, 9, 4))
    draws, info, draw_info = BasicSolver.batch_sample(flatten(kernel), params, xk, sigk, rk, xs, madd, z, 0.0)
    outcomes = set()
    for b in range(nb):
        p0 = kernel.get_parameter_vector(include_frozen=True)
        kernel.set_parameter_vector(params[b], include_frozen=True)
        try:
            BasicSolver(kernel).compute(xk, sigk[b])
            k_ok = True
        except np.linalg.LinAlgError as e:
            k_ok = False
            assert info[b] == _minor(e), (b, info[b], str(e))
        finally:
            kernel.set_parameter_vector(p0, include_frozen=True)
        if not k_ok:
            assert draw_info[b] == 0 and np.all(np.isnan(draws[b]))
            outcomes.add("k")
            continue
        assert info[b] == 0
        want = _single(kernel, params[b], xk, sigk[b], rk[b], xs, madd[b], z[b], 0.0)
        if isinstance(want, Exception):
            assert draw_info[b] == _minor(want) and np.all(np.isnan(draws[b])), (b, draw_info[b], str(want))
            outcomes.add("cov")
        else:
            assert draw_info[b] == 0 and np.array_equal(draws[b], want), b
            outcomes.add("ok")
    assert outcomes == {"k", "cov", "ok"}, outcomes


def test_loop_routes_give_the_loops_draws(gpu):
    import george_b200 as george
    from george_b200 import kernels
    rng = np.random.default_rng(15)
    x = np.sort(rng.uniform(0, 10, 400))
    y = np.sin(x) + 0.1 * rng.standard_normal(400)
    t = np.linspace(-1, 11, 50)

    class NoBatch(george.BasicSolver):
        batch_sample = None

    gph = george.GP(1.0 * kernels.ExpSquaredKernel(1.0), solver=george.HODLRSolver, tol=1e-12, min_size=50)
    gpn = george.GP(1.0 * kernels.ExpSquaredKernel(1.0), solver=NoBatch)
    for gp in (gph, gpn):
        gp.compute(x, 0.1)
        vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((3, len(gp)))
        for size in (1, 9):
            gp.log_likelihood(y)
            st = _state(gp)
            g1, g2 = np.random.default_rng(size), np.random.default_rng(size)
            got = gp.batch_sample_conditional(vecs, y, t, size, rng=g1, jitter=1e-6)
            _assert_state(gp, st)
            assert np.array_equal(got, _loop(gp, vecs, y, t, size, rng=g2, jitter=1e-6))
            assert _same_gen(g1, g2)

    gpd = george.GP(1.0 * kernels.ExpSquaredKernel(1.0))
    gpd.compute(x, 0.1)
    vecs = gpd.get_parameter_vector() + 0.05 * rng.standard_normal((3, len(gpd)))
    t = np.linspace(-1, 11, 12)
    gpd.log_likelihood(y)
    st = _state(gpd)
    np.random.seed(4)
    with _nowarn():
        got = gpd.batch_sample_conditional(vecs, y, t, 2)
    _assert_state(gpd, st)
    np.random.seed(4)
    with _nowarn():
        want = _loop(gpd, vecs, y, t, 2)
    assert np.array_equal(got, want)


class _nowarn(object):
    """Silence numpy's warning about a covariance that is not positive semi-definite on the host route."""

    def __enter__(self):
        import warnings
        self._cm = warnings.catch_warnings()
        self._cm.__enter__()
        warnings.simplefilter("ignore", RuntimeWarning)

    def __exit__(self, *a):
        return self._cm.__exit__(*a)


def test_pickled_gp_gives_the_same_draws(gpu):
    import george_b200 as george
    from george_b200 import kernels
    rng = np.random.default_rng(17)
    x = np.sort(rng.uniform(0, 10, 300))
    y = np.sin(x) + 0.1 * rng.standard_normal(300)
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0), mean=0.3, fit_mean=True)
    gp.compute(x, 0.1)
    gp.log_likelihood(y)
    vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((4, len(gp)))
    t = np.linspace(0, 10, 40)
    want = gp.batch_sample_conditional(vecs, y, t, 8, rng=np.random.default_rng(3), jitter=1e-6)
    gp2 = pickle.loads(pickle.dumps(gp))
    assert np.array_equal(gp2.batch_sample_conditional(vecs, y, t, 8, rng=np.random.default_rng(3), jitter=1e-6),
                          want)


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
    draws = gp.batch_sample_conditional(vecs, y, t, 64, rng=np.random.default_rng(8), jitter=1e-6)
    assert draws.shape == (32, 64, 500) and np.all(np.isfinite(draws))
    # in the loop, member b draws from the generator after the b members before it
    for b in (0, 9, 20, 31):
        g = np.random.default_rng(8)
        for _ in range(b):
            g.standard_normal((64, 500))
        gp.set_parameter_vector(vecs[b])
        assert np.array_equal(draws[b], gp.sample_conditional(y, t, 64, rng=g, jitter=1e-6)), b
