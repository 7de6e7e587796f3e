# -*- coding: utf-8 -*-
"""GP.batch_loo_predict, GP.batch_loo_log_likelihood, GP.batch_grad_loo_log_likelihood and
BasicSolver.batch_loo_terms on the device: every member's alpha, d, beta, g and diag are the single path's (compute +
loo_terms) bit for bit, the GP-level results are the per-vector loops' bit for bit, failures stay with their member,
the value and gradient agree with the longdouble LOO formula, the results do not depend on B, the position or the
chunking, and the launch count does not grow with B."""
import numpy as np
import pytest
from numpy.linalg import LinAlgError

import test_gpu_batch_grad as bg
import test_gpu_loo as tl

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _free_batch_workspace():
    """The process-wide batch workspace grows to this module's largest call (n = 4096: about 4 GB with A); free it
    afterwards so that the tests after this module start from the device memory they would have had without it."""
    yield
    import gc
    from george_b200.solvers import basic
    basic._batch_handle = None
    gc.collect()

# bars: 50-70x the largest value measured on one H100 80GB HBM3 (SXM, 700 W power limit), as tests/test_gpu_loo.py's
VALUE_TOL = 2e-13   # value vs the longdouble formula, relative                            (measured 4.0e-15)
GRAD_TOL = 5e-13    # gradient vs the longdouble formula, per entry over its |terms| scale   (measured 7.5e-15)


def _single(kernel, p, x, sig, r, which):
    """GP.grad_loo_log_likelihood's device steps for one member: compute, loo_terms (pass 1 and both passes)."""
    from george_b200 import BasicSolver
    p0 = kernel.get_parameter_vector(include_frozen=True)
    kernel.set_parameter_vector(p, include_frozen=True)
    try:
        s = BasicSolver(kernel)
        s.compute(x, sig)
        return s.loo_terms(r), s.loo_terms(r, which)
    finally:
        kernel.set_parameter_vector(p0, include_frozen=True)


def _check_members(kernel, ndim, n, nb=3):
    from george_b200 import BasicSolver
    from george_b200._spec import flatten
    spec, which = flatten(kernel), bg._which(kernel)
    params = bg._perturbed(kernel, nb, n)
    x, sig, r = bg._inputs(n, ndim, nb, n + 1)
    a1, d1, info1 = BasicSolver.batch_loo_terms(spec, params, x, sig, r)
    alpha, d, beta, g, diag, info = BasicSolver.batch_loo_terms(spec, params, x, sig, r, which)
    assert np.all(info == 0) and np.all(info1 == 0), (n, info, info1)
    assert np.array_equal(a1, alpha) and np.array_equal(d1, d), n
    for b in range(nb):
        (sa, sd), (ga, gd, gbeta, gg, gdiag) = _single(kernel, params[b], x, sig[b], r[b], which)
        assert np.array_equal(sa, ga) and np.array_equal(sd, gd)
        for got, want, what in ((alpha, ga, "alpha"), (d, gd, "d"), (beta, gbeta, "beta"), (g, gg, "g"),
                                (diag, gdiag, "diag")):
            assert np.array_equal(got[b], want), (n, b, what, np.max(np.abs(got[b] - want)))


@pytest.mark.parametrize("name", [z[0] for z in bg._zoo()])
def test_members_match_the_single_path(gpu, name):
    _, kernel, ndim = [z for z in bg._zoo() if z[0] == name][0]
    for n in bg.SIZES:
        _check_members(kernel, ndim, n)


@pytest.mark.parametrize("n", [2048, 2049])
def test_members_match_the_single_path_either_side_of_the_single_slice_product(gpu, n):
    """From n = 2049 the G^T G product of a 132-SM H100 runs in one split-K slice, below it in several."""
    from george_b200 import kernels
    _check_members(1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3), 3, n, nb=2)


# ---- the GP layer ----------------------------------------------------------------------------------------------------

def _loop(gp, vecs, y, kind, quiet=False):
    """The per-vector path each batch method stands for: (mu, var), the values, or (values, gradients)."""
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
    return got.shape == want.shape and np.array_equal(got, want)


KINDS = ["predict", "value", "grad"]


def _check_gp(gp, y, vecs, quiet=False, kinds=KINDS):
    """The methods of ``kinds`` against their loops, bit for bit, the GP left as it was; the batch results by kind."""
    out = {}
    for kind in kinds:
        gp.log_likelihood(y)
        st = bg._state(gp)
        got = _batch(gp, vecs, y, kind, quiet)
        bg._assert_state(gp, st)
        want = _loop(gp, vecs, y, kind, quiet)
        assert _same(got, want), kind
        out[kind] = got
    if "value" in out and "grad" in out:
        assert np.array_equal(out["value"], out["grad"][0])
    gp.log_likelihood(y)  # (the reference loop above left the GP at another factorisation)
    return out


def test_co2(gpu):
    gp, y = bg._co2_gp()
    rng = np.random.default_rng(5)
    vecs = gp.get_parameter_vector() + 1e-4 * rng.standard_normal((6, len(gp)))
    out = _check_gp(gp, y, vecs)
    assert np.all(np.isfinite(out["grad"][0])) and np.all(np.isfinite(out["grad"][1]))


def test_matern52_3d(gpu):
    import george_b200 as george
    from george_b200 import kernels
    rng = np.random.default_rng(21)
    x = rng.uniform(-3, 3, (400, 3))
    y = np.sin(x[:, 0]) * np.cos(x[:, 1]) + 0.1 * rng.standard_normal(400)
    gp = george.GP(1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3), white_noise=np.log(0.05),
                   fit_white_noise=True)
    gp.compute(x, 0.3)
    _check_gp(gp, y, gp.get_parameter_vector() + 0.05 * rng.standard_normal((5, len(gp))))


def test_user_kernel(gpu):
    import george_b200 as george
    from george_b200 import kernels
    rng = np.random.default_rng(22)
    x = rng.uniform(0, 3, (150, 2))
    y = np.sin(2 * x[:, 0]) + 0.1 * rng.standard_normal(150)
    gp = george.GP(0.8 * kernels.CauchyKernel(metric=0.7, ndim=2), mean=0.1, fit_mean=True)
    gp.compute(x, 0.1)
    _check_gp(gp, y, gp.get_parameter_vector() + 0.05 * rng.standard_normal((4, len(gp))))


def test_fitted_mean_non_constant_white_noise_and_frozen_parameters(gpu):
    import george_b200 as george
    from george_b200 import kernels
    from george_b200.modeling import Model

    class LineMean(Model):
        parameter_names = ("m", "b")

        def get_value(self, t):
            return t.flatten() * self.m + self.b

        def compute_gradient(self, t):
            t = t.flatten()
            return np.vstack([t, np.ones_like(t)])

    class LinearNoise(Model):
        parameter_names = ("c", "s")

        def get_value(self, t):
            return self.c + self.s * t.flatten()

        def compute_gradient(self, t):
            t = t.flatten()
            return np.vstack([np.ones_like(t), t])

    rng = np.random.default_rng(23)
    t = np.sort(rng.uniform(0, 4, 250))
    y = 0.3 * t + np.cos(2 * t) + 0.1 * rng.standard_normal(250)
    gp = george.GP(1.2 * kernels.ExpSquaredKernel(0.6) + 0.3 * kernels.Matern32Kernel(2.0),
                   mean=LineMean(m=0.3, b=0.0), fit_mean=True,
                   white_noise=LinearNoise(c=np.log(0.05), s=0.2), fit_white_noise=True)
    gp.compute(t, 0.02)
    vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((5, len(gp)))
    _check_gp(gp, y, vecs)
    for name in ("mean:b", "white_noise:s", "kernel:k1:k1:log_constant"):
        gp.freeze_parameter(name)
    vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((5, len(gp)))
    out = _check_gp(gp, y, vecs)
    assert out["grad"][1].shape == (5, len(gp)) == (5, 5)
    assert gp.mean.get_parameter_vector(include_frozen=True)[1] == 0.0


def _check_failures(gp, y, vecs, bad, exc_type):
    """quiet: the loops' results, the bad members -inf with zero gradients; otherwise the loops' first exception."""
    for kind in ("value", "grad"):
        got = _check_gp(gp, y, vecs, quiet=True, kinds=[kind])[kind]
        value = got if kind == "value" else got[0]
        assert np.all(np.isneginf(value[bad])) and np.all(np.isfinite(np.delete(value, bad)))
        if kind == "grad":
            assert np.all(got[1][bad] == 0.0)
    for kind in KINDS:
        gp.log_likelihood(y)
        st = bg._state(gp)
        with pytest.raises(exc_type) as batch_exc:
            _batch(gp, vecs, y, kind)
        bg._assert_state(gp, st)
        with pytest.raises(exc_type) as loop_exc:
            _loop(gp, vecs, y, kind)
        assert type(batch_exc.value) is type(loop_exc.value)
        assert str(batch_exc.value) == str(loop_exc.value)


def test_not_positive_definite_members(gpu):
    gp, y = bg._dot_gp()
    vecs = np.full((8, len(gp)), np.log(0.1))
    bad = [2, 5]
    vecs[bad, 0] = -80.0  # K = x x^T + 1.8e-35 I: rank one, not positive definite
    _check_failures(gp, y, vecs, bad, LinAlgError)


def test_non_finite_mean_member(gpu):
    gp, y = bg._co2_gp(n=120)
    rng = np.random.default_rng(8)
    vecs = gp.get_parameter_vector() + 1e-4 * rng.standard_normal((6, len(gp)))
    vecs[3, 0] = np.nan
    _check_failures(gp, y, vecs, [3], ValueError)


def test_hodlr_takes_the_loop(gpu):
    import george_b200 as george
    from george_b200 import kernels
    rng = np.random.default_rng(15)
    x = np.sort(rng.uniform(0, 10, 400))
    y = np.sin(x) + 0.1 * rng.standard_normal(400)
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0), white_noise=np.log(0.01), fit_white_noise=True,
                   solver=george.HODLRSolver, tol=1e-12, min_size=50)
    gp.compute(x, 0.1)
    _check_gp(gp, y, gp.get_parameter_vector() + 0.05 * rng.standard_normal((3, len(gp))))


def test_accuracy_against_the_longdouble_formula(gpu, record_property):
    """(value, grad) of every member against test_gpu_loo's longdouble formula on the member's K, with a fitted
    constant mean and white noise: mean part sum(beta), white-noise part exp(wn) sum(diag A), kernel part
    einsum(dK, A)."""
    import george_b200 as george
    from george_b200 import kernels
    kernel, ndim = tl._dense_kernels()["m52_3d_axis"]
    x, yerr, y = tl._inputs(257, ndim)
    gp = george.GP(kernel, mean=0.1, fit_mean=True, white_noise=np.log(0.01), fit_white_noise=True)
    gp.compute(x, yerr)
    rng = np.random.default_rng(24)
    vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((3, len(gp)))
    value, grad = gp.batch_grad_loo_log_likelihood(vecs, y, return_value=True)
    p0 = gp.get_parameter_vector()
    errs = {"value": 0.0, "grad": 0.0}
    try:
        for b, v in enumerate(vecs):
            gp.set_parameter_vector(v)
            wn = np.exp(gp.white_noise.get_value(x))
            K = tl._kmat(gp.kernel, x, np.sqrt(yerr ** 2 + wn))
            ref = tl._ld_formula(K, y - gp.mean.get_value(x), gp.kernel.get_gradient(x, include_frozen=True))
            dA = np.diag(ref["A"])
            want = np.concatenate([[np.sum(ref["beta"])], [np.sum(wn * dA)], ref["g"]])
            scale = np.concatenate([[np.sum(np.abs(ref["beta"]))], [np.sum(np.abs(wn * dA))], ref["gscale"]])
            errs["value"] = max(errs["value"], float(abs(value[b] - ref["value"]) / abs(ref["value"])))
            errs["grad"] = max(errs["grad"], float(np.max(np.abs(grad[b] - want) / scale)))
    finally:
        gp.set_parameter_vector(p0)
    record_property("batch_loo_err", errs)
    assert errs["value"] <= VALUE_TOL and errs["grad"] <= GRAD_TOL, errs


# ---- position, chunking, launches, a large batch ----------------------------------------------------------------------

def test_results_do_not_depend_on_batch_position_or_chunking(gpu, monkeypatch):
    from george_b200 import BasicSolver, kernels
    from george_b200._spec import flatten
    kernel = 1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3)
    spec, which = flatten(kernel), bg._which(kernel)
    n, nb = 130, 12
    params = bg._perturbed(kernel, nb, 11)
    x, sig, r = bg._inputs(n, 3, nb, 12)
    monkeypatch.delenv("BGP_BATCH_CHUNK", raising=False)
    for w in (None, which):
        ref = BasicSolver.batch_loo_terms(spec, params, x, sig, r, w)

        def same(got, idx_got, idx_ref):
            return all(np.array_equal(a[idx_got], b[idx_ref]) for a, b in zip(got, ref))

        assert same(BasicSolver.batch_loo_terms(spec, params, x, sig, r, w), slice(None), slice(None))
        for b in (0, 5, 11):
            one = BasicSolver.batch_loo_terms(spec, params[b:b + 1], x, sig[b:b + 1], r[b:b + 1], w)
            assert same(one, 0, b), b
        order = [i for i in range(nb) if i != 5] + [5]
        assert same(BasicSolver.batch_loo_terms(spec, params[order], x, sig[order], r[order], w), -1, 5)
        for chunk in ("1", "5", "64"):  # 5: two chunks of five and a ragged tail of two
            monkeypatch.setenv("BGP_BATCH_CHUNK", chunk)
            got = BasicSolver.batch_loo_terms(spec, params, x, sig, r, w)
            monkeypatch.delenv("BGP_BATCH_CHUNK")
            assert same(got, slice(None), slice(None)), chunk


def test_launch_count_does_not_grow_with_the_batch(gpu, monkeypatch):
    from george_b200 import BasicSolver, _lib, kernels
    from george_b200._spec import flatten
    monkeypatch.delenv("BGP_BATCH_CHUNK", raising=False)
    lib = _lib.load()
    kernel = 1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3)
    spec, which = flatten(kernel), bg._which(kernel)
    n = 1000
    params = bg._perturbed(kernel, 48, 13)
    x, sig, r = bg._inputs(n, 3, 48, 14)
    for w in (None, which):
        counts = []
        for nb in (1, 48):
            c0 = lib.bgp_launch_count()
            BasicSolver.batch_loo_terms(spec, params[:nb], x, sig[:nb], r[:nb], w)
            counts.append(lib.bgp_launch_count() - c0)
        assert counts[0] == counts[1] > 0, (w, counts)


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
    value, grad = gp.batch_grad_loo_log_likelihood(vecs, y, return_value=True)
    pick = [0, 9, 20, 31]
    assert np.all(np.isfinite(value)) and np.all(np.isfinite(grad))
    want = _loop(gp, vecs[pick], y, "grad")
    assert np.array_equal(value[pick], want[0]) and np.array_equal(grad[pick], want[1])
    mu, var = gp.batch_loo_predict(vecs, y)
    want = _loop(gp, vecs[pick], y, "predict")
    assert np.array_equal(mu[pick], want[0]) and np.array_equal(var[pick], want[1])
