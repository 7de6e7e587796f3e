# -*- coding: utf-8 -*-
"""GP.batch_grad_log_likelihood / BasicSolver.batch_grad_terms on the device: every member's alpha, g, diag and
log-determinant are the single path's (compute + grad_terms) bit for bit, the GP-level gradients are the per-vector
loop's bit for bit, failures stay with their member, the results do not depend on B, the position or the chunking,
and the launch count does not grow with B."""
import pickle

import numpy as np
import pytest

import hiprec

pytestmark = pytest.mark.gpu

SIZES = [1, 2, 7, 8, 9, 63, 64, 65, 129, 300, 1000]   # 8 | 9: either side of the few-column solve of K^-1


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


def _which(kernel):
    """Every parameter but the last (when there are two or more): the zeros of g are exercised too."""
    w = np.ones(len(kernel.get_parameter_vector(include_frozen=True)), dtype=np.uint32)
    if len(w) > 1:
        w[-1] = 0
    return w


def _single(kernel, p, x, sig, r, which):
    """GP.grad_log_likelihood's device steps for one member: compute, grad_terms."""
    from george_b200 import BasicSolver
    p0 = kernel.get_parameter_vector(include_frozen=True)
    kernel.set_parameter_vector(p, include_frozen=True)
    try:
        s = BasicSolver(kernel)
        s.compute(x, sig)
        alpha, g, diag = s.grad_terms(r, which)
        return s.log_determinant, alpha, g, diag
    finally:
        kernel.set_parameter_vector(p0, include_frozen=True)


@pytest.mark.parametrize("name", [z[0] for z in _zoo()])
def test_members_match_the_single_path(gpu, name):
    from george_b200 import BasicSolver
    from george_b200._spec import flatten
    _, kernel, ndim = [z for z in _zoo() if z[0] == name][0]
    spec, which = flatten(kernel), _which(kernel)
    for n in SIZES:
        params = _perturbed(kernel, 3, n)
        x, sig, r = _inputs(n, ndim, 3, n + 1)
        ld, q, alpha, g, diag, info = BasicSolver.batch_grad_terms(spec, params, x, sig, r, which)
        assert np.all(info == 0), (name, n, info)
        _, q_ll, _ = BasicSolver.batch_log_likelihood(spec, params, x, sig, r)
        assert np.array_equal(q, q_ll), (name, n)
        for b in range(3):
            ld1, a1, g1, d1 = _single(kernel, params[b], x, sig[b], r[b], which)
            assert ld[b] == ld1, (name, n, b)
            assert np.array_equal(alpha[b], a1), (name, n, b, np.max(np.abs(alpha[b] - a1)))
            assert np.array_equal(g[b], g1), (name, n, b, g[b], g1)
            assert np.array_equal(diag[b], d1), (name, n, b, np.max(np.abs(diag[b] - d1)))


@pytest.mark.parametrize("n", [65, 700])
def test_accuracy_against_extended_precision(gpu, oracle, n):
    """g and diag against K^-1 from a longdouble Cholesky and the oracle's gradient tensor, with the bars of
    tests/test_gpu_ops.py::test_grad_terms_match_host_composition."""
    from george_b200 import BasicSolver, kernels
    from george_b200._spec import flatten, patch_specs
    kernel = 0.7 * kernels.Matern52Kernel([0.3, 0.6], ndim=2) + 0.2 * kernels.ExpSquaredKernel(0.1, ndim=2, axes=0)
    spec = flatten(kernel)
    rng = np.random.default_rng(n)
    x = rng.uniform(0, 1, (n, 2))
    params = _perturbed(kernel, 3, 3 * n)
    sig = 0.1 + 0.05 * rng.uniform(size=(3, n))
    r = np.sin(4 * x[:, 0]) + x[:, 1] + 0.1 * rng.standard_normal((3, n))
    which = np.ones(params.shape[1], dtype=np.uint32)
    _, _, alpha, g, diag, info = BasicSolver.batch_grad_terms(spec, params, x, sig, r, which)
    assert np.all(info == 0)
    for b, ms in enumerate(patch_specs(spec, params)):
        K = oracle.value_symmetric(ms, x) + np.diag(sig[b] ** 2)
        Kinv = hiprec.solve_ld(hiprec.chol_ld(K), np.eye(n))
        a_ref = Kinv @ r[b].astype(hiprec.LD)
        A = np.outer(a_ref, a_ref) - Kinv
        dK = oracle.gradient_general(ms, which, x, x)
        ref = np.einsum("ijk,ij", dK.astype(hiprec.LD), A)
        scale = np.einsum("ijk,ij", np.abs(dK), np.abs(A).astype(np.float64))
        assert np.linalg.norm((alpha[b] - a_ref).astype(np.float64)) <= 1e-8 * np.linalg.norm(a_ref.astype(np.float64))
        assert np.all(np.abs((g[b] - ref).astype(np.float64)) <= 1e-7 * scale), (b, g[b], ref)
        dref = np.diag(A)
        assert np.linalg.norm((diag[b] - dref).astype(np.float64)) <= 1e-7 * np.linalg.norm(dref.astype(np.float64))


def _co2_gp(n=300, seed=0):
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
            gp.kernel.dirty, gp._const)


def _assert_state(gp, st):
    now = _state(gp)
    assert np.array_equal(st[0], now[0])
    assert now[1] == st[1] and now[5] == st[5] and now[6] == st[6]
    assert now[2] is st[2] and now[3] is st[3] and now[4] is st[4]


def _loop(gp, vecs, y, quiet=False, return_ll=False):
    """The per-vector path batch_grad_log_likelihood stands for."""
    p0 = gp.get_parameter_vector()
    ll = np.empty(len(vecs))
    grad = np.empty((len(vecs), len(gp)))
    try:
        for b, v in enumerate(vecs):
            gp.set_parameter_vector(v)
            if return_ll:
                ll[b] = gp.log_likelihood(y, quiet=quiet)
            grad[b] = gp.grad_log_likelihood(y, quiet=quiet)
    finally:
        gp.set_parameter_vector(p0)
    return (ll, grad) if return_ll else grad


def _close(a, b):
    return np.all((a == b) | (np.abs(a - b) <= 1e-12 * np.maximum(1.0, np.abs(b))))


def _check_gp(gp, y, vecs, quiet=False):
    gp.log_likelihood(y)
    st = _state(gp)
    got = gp.batch_grad_log_likelihood(vecs, y, quiet=quiet)
    _assert_state(gp, st)
    ll, got2 = gp.batch_grad_log_likelihood(vecs, y, quiet=quiet, return_log_likelihood=True)
    _assert_state(gp, st)
    assert np.array_equal(got, got2)
    assert np.array_equal(ll, gp.batch_log_likelihood(vecs, y, quiet=quiet))
    _assert_state(gp, st)
    want = _loop(gp, vecs, y, quiet=quiet)
    assert np.array_equal(got, want), np.max(np.abs(got - want))
    ll_loop, want2 = _loop(gp, vecs, y, quiet=quiet, return_ll=True)
    assert np.array_equal(got2, want2)
    assert _close(ll, ll_loop), np.max(np.abs(ll - ll_loop))
    gp.log_likelihood(y)  # (the reference loop above left the GP at another factorisation)
    return ll, got


def test_co2_gradients(gpu):
    gp, y = _co2_gp()
    rng = np.random.default_rng(5)
    vecs = gp.get_parameter_vector() + 1e-4 * rng.standard_normal((6, len(gp)))
    ll, grad = _check_gp(gp, y, vecs)
    assert np.all(np.isfinite(ll)) and np.all(np.isfinite(grad))


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
    gp = george.GP(0.5 * kernels.Matern32Kernel(1.5), mean=PolynomialModel(m=0.4, b=0.0),
                   white_noise=np.log(0.1 ** 2), fit_white_noise=True)
    gp.freeze_parameter("mean:b")
    gp.compute(t, 0.05)
    vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((5, len(gp)))
    _check_gp(gp, y, vecs)
    assert np.array_equal(gp.mean.get_parameter_vector(include_frozen=True), [0.4, 0.0])


def test_non_constant_white_noise(gpu):
    import george_b200 as george
    from george_b200 import kernels
    from george_b200.modeling import Model

    class LinearNoise(Model):
        parameter_names = ("c", "s")

        def get_value(self, t):
            return self.c + self.s * t.flatten()

    rng = np.random.default_rng(7)
    t = np.sort(rng.uniform(0, 4, 200))
    y = np.cos(2 * t) + 0.1 * rng.standard_normal(200)
    gp = george.GP(1.2 * kernels.ExpSquaredKernel(0.6), mean=0.1, fit_mean=True,
                   white_noise=LinearNoise(c=np.log(0.05), s=0.2), fit_white_noise=True)
    gp.compute(t, 0.02)
    vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((5, len(gp)))
    _check_gp(gp, y, vecs)
    assert np.array_equal(gp.white_noise.get_parameter_vector(include_frozen=True), [np.log(0.05), 0.2])


def _dot_gp():
    import george_b200 as george
    from george_b200 import kernels
    x = np.linspace(0.1, 1, 50)
    gp = george.GP(kernels.DotProductKernel(), white_noise=np.log(0.1), fit_white_noise=True)
    gp.compute(x, 0.0)
    y = np.cos(x)
    return gp, y


def _check_failures(gp, y, vecs, bad, exc_type, value_fails=True):
    """quiet: the loop's values, the bad members' gradients zero (and their values -inf when the value fails too);
    otherwise the loop's first exception."""
    for return_ll in (False, True):
        gp.log_likelihood(y)
        st = _state(gp)
        got = gp.batch_grad_log_likelihood(vecs, y, quiet=True, return_log_likelihood=return_ll)
        _assert_state(gp, st)
        want = _loop(gp, vecs, y, quiet=True, return_ll=return_ll)
        if return_ll:
            assert np.array_equal(got[1], want[1])
            assert _close(got[0], want[0]) and np.all(np.isneginf(got[0][bad]) == value_fails)
            got = got[1]
        else:
            assert np.array_equal(got, want)
        assert np.all(got[bad] == 0.0)
        gp.log_likelihood(y)
        st = _state(gp)
        with pytest.raises(exc_type) as batch_exc:
            gp.batch_grad_log_likelihood(vecs, y, return_log_likelihood=return_ll)
        _assert_state(gp, st)
        with pytest.raises(exc_type) as loop_exc:
            _loop(gp, vecs, y, return_ll=return_ll)
        assert type(batch_exc.value) is type(loop_exc.value)
        assert str(batch_exc.value) == str(loop_exc.value)


def test_failures_stay_with_their_member(gpu):
    from george_b200 import BasicSolver
    from george_b200._spec import flatten
    gp, y = _dot_gp()
    vecs = np.full((8, len(gp)), np.log(0.1))
    bad = [2, 5]
    vecs[bad, 0] = -80.0  # K = x x^T + 1.8e-35 I: rank one, not positive definite
    _check_failures(gp, y, vecs, bad, np.linalg.LinAlgError)

    # through the ABI: the good members are the single path's, the bad ones NaN with the single path's minor index
    x = gp._x
    sig = np.sqrt(np.zeros((8, 50)) + np.exp(vecs[:, :1]))
    r = np.tile(y, (8, 1))
    which = np.zeros(0, dtype=np.uint32)
    ld, q, alpha, g, diag, info = BasicSolver.batch_grad_terms(flatten(gp.kernel), np.zeros((8, 0)), x, sig, r, which)
    assert g.shape == (8, 0)
    for b in range(8):
        if b in bad:
            with pytest.raises(np.linalg.LinAlgError) as e:
                BasicSolver(gp.kernel).compute(x, sig[b])
            assert info[b] > 0 and str(e.value).startswith("%d-th" % info[b])
            assert np.isnan(ld[b]) and np.isnan(q[b]) and np.all(np.isnan(alpha[b])) and np.all(np.isnan(diag[b]))
        else:
            assert info[b] == 0
            ld1, a1, _, d1 = _single(gp.kernel, np.zeros(0), x, sig[b], r[b], which)
            assert ld[b] == ld1 and np.array_equal(alpha[b], a1) and np.array_equal(diag[b], d1)


def test_non_finite_mean_member(gpu):
    gp, y = _co2_gp(n=120)
    rng = np.random.default_rng(8)
    vecs = gp.get_parameter_vector() + 1e-4 * rng.standard_normal((6, len(gp)))
    vecs[3, 0] = np.nan
    _check_failures(gp, y, vecs, [3], ValueError)


def _np65_kernel():
    """1 + 36 + 1 + 21 + 1 + 5 = 65 parameters, 8-D: one more than the device contraction takes."""
    from george_b200 import kernels as K

    def general(nax, seed, scale):
        a = np.random.default_rng(seed).normal(size=(nax, nax))
        return scale * (np.eye(nax) + 0.2 * a @ a.T / nax)

    return (1.0 * K.ExpSquaredKernel(general(8, 3, 8.0), ndim=8)
            + 0.5 * K.ExpSquaredKernel(general(6, 4, 6.0), ndim=8, axes=list(range(6)))
            + 0.3 * K.Matern32Kernel([1.0, 2.0, 3.0, 4.0, 5.0], ndim=8, axes=[3, 4, 5, 6, 7]))


def test_more_than_64_kernel_parameters(gpu):
    import george_b200 as george
    from george_b200 import BasicSolver
    from george_b200._spec import flatten
    kernel = _np65_kernel()
    assert kernel.full_size == 65
    rng = np.random.default_rng(9)
    x = rng.uniform(-1, 1, (150, 8))
    y = np.sin(x[:, 0])
    gp = george.GP(kernel, mean=0.0, fit_mean=True, white_noise=np.log(0.1), fit_white_noise=True)
    gp.compute(x, 0.1)
    vecs = gp.get_parameter_vector() + 1e-3 * rng.standard_normal((4, len(gp)))
    _check_failures(gp, y, vecs, [0, 1, 2, 3], ValueError, value_fails=False)
    ll, _ = gp.batch_grad_log_likelihood(vecs, y, quiet=True, return_log_likelihood=True)
    assert np.all(np.isfinite(ll)) and np.array_equal(ll, gp.batch_log_likelihood(vecs, y))
    with pytest.raises(ValueError, match="64"):
        BasicSolver.batch_grad_terms(flatten(kernel), np.tile(kernel.get_parameter_vector(include_frozen=True), (2, 1)),
                                     x, np.ones((2, 150)), np.ones((2, 150)), np.ones(65, dtype=np.uint32))


def test_results_do_not_depend_on_batch_position_or_chunking(gpu, monkeypatch):
    from george_b200 import BasicSolver, kernels
    from george_b200._spec import flatten
    kernel = 1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3)
    spec, which = flatten(kernel), _which(kernel)
    n, nb = 130, 12
    params = _perturbed(kernel, nb, 11)
    x, sig, r = _inputs(n, 3, nb, 12)
    monkeypatch.delenv("BGP_BATCH_CHUNK", raising=False)
    ref = BasicSolver.batch_grad_terms(spec, params, x, sig, r, which)

    def same(got, idx_got, idx_ref):
        return all(np.array_equal(a[idx_got], b[idx_ref]) for a, b in zip(got, ref))

    assert same(BasicSolver.batch_grad_terms(spec, params, x, sig, r, which), slice(None), slice(None))
    for b in (0, 5, 11):
        one = BasicSolver.batch_grad_terms(spec, params[b:b + 1], x, sig[b:b + 1], r[b:b + 1], which)
        assert same(one, 0, b), b
    order = [i for i in range(nb) if i != 5] + [5]
    assert same(BasicSolver.batch_grad_terms(spec, params[order], x, sig[order], r[order], which), -1, 5)
    for chunk in ("1", "5", "64"):
        monkeypatch.setenv("BGP_BATCH_CHUNK", chunk)
        got = BasicSolver.batch_grad_terms(spec, params, x, sig, r, which)
        monkeypatch.delenv("BGP_BATCH_CHUNK")
        assert same(got, slice(None), slice(None)), chunk


def test_launch_count_does_not_grow_with_the_batch(gpu, monkeypatch):
    from george_b200 import BasicSolver, _lib, kernels
    from george_b200._spec import flatten
    monkeypatch.delenv("BGP_BATCH_CHUNK", raising=False)
    lib = _lib.load()
    kernel = 1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3)
    spec, which = flatten(kernel), _which(kernel)
    n = 1000
    params = _perturbed(kernel, 48, 13)
    x, sig, r = _inputs(n, 3, 48, 14)
    counts = []
    for nb in (1, 48):
        c0 = lib.bgp_launch_count()
        BasicSolver.batch_grad_terms(spec, params[:nb], x, sig[:nb], r[:nb], which)
        counts.append(lib.bgp_launch_count() - c0)
    assert counts[0] == counts[1] > 0, counts


def test_hodlr_and_trivial_take_the_loop_and_gp_pickles(gpu):
    import george_b200 as george
    from george_b200 import kernels
    rng = np.random.default_rng(15)
    x = np.sort(rng.uniform(0, 10, 400))
    y = np.sin(x) + 0.1 * rng.standard_normal(400)
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0), white_noise=np.log(0.01), fit_white_noise=True,
                   solver=george.HODLRSolver, tol=1e-12, min_size=50)
    gp.compute(x, 0.1)
    vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((3, len(gp)))
    _check_gp(gp, y, vecs)

    gpt = george.GP(mean=0.3, fit_mean=True, white_noise=np.log(0.2))
    assert gpt.solver_type is george.TrivialSolver
    gpt.compute(x, 0.05)
    vt = gpt.get_parameter_vector() + 0.05 * rng.standard_normal((3, len(gpt)))
    st = _state(gpt)
    got = gpt.batch_grad_log_likelihood(vt, y)
    _assert_state(gpt, st)
    assert np.array_equal(got, _loop(gpt, vt, y))

    gpd = george.GP(1.0 * kernels.ExpSquaredKernel(1.0), white_noise=np.log(0.01), fit_white_noise=True)
    gpd.compute(x, 0.1)
    gpd.log_likelihood(y)
    want = gpd.batch_grad_log_likelihood(vecs, y, return_log_likelihood=True)
    gp2 = pickle.loads(pickle.dumps(gpd))
    got = gp2.batch_grad_log_likelihood(vecs, y, return_log_likelihood=True)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    assert np.array_equal(want[1], _loop(gpd, vecs, y))


def test_large_batch(gpu):
    import george_b200 as george
    from george_b200 import kernels
    rng = np.random.default_rng(16)
    n = 4096
    x = rng.uniform(-3, 3, (n, 3))
    y = np.sin(x[:, 0]) * np.cos(x[:, 1]) + 0.1 * rng.standard_normal(n)
    gp = george.GP(1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3), white_noise=np.log(0.05),
                   fit_white_noise=True)
    gp.compute(x, 0.3)
    vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((32, len(gp)))
    ll, grad = gp.batch_grad_log_likelihood(vecs, y, return_log_likelihood=True)
    pick = [0, 9, 20, 31]
    assert np.all(np.isfinite(ll)) and np.all(np.isfinite(grad))
    assert np.array_equal(grad[pick], _loop(gp, vecs[pick], y))
