# -*- coding: utf-8 -*-
"""GP.batch_fisher_information / BasicSolver.batch_fisher_terms on the device: every member's rows, diagonals, mean
solve and gradient terms are the single path's (compute + fisher_terms + apply_inverse) bit for bit, the GP-level
results are the per-vector loop's bit for bit, F agrees with test_gpu_fisher's longdouble brute force and is exactly
symmetric and PSD, failures stay with their member, the results do not depend on B, the position or the chunking, and
the launch count does not grow with B."""
import numpy as np
import pytest
from numpy.linalg import LinAlgError

import test_gpu_batch_grad as bg
import test_gpu_fisher as tf

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _free_batch_workspace():
    """The process-wide batch workspace grows to this module's largest call (n = 4096: factor, K^-1, P and T of up to
    eight members, about 4 GB); free it afterwards so that the tests after this module start from the device memory
    they would have had without it."""
    yield
    import gc
    from george_b200.solvers import basic
    basic._batch_handle = None
    gc.collect()


NV, NM = 2, 2  # white-noise vectors and mean gradients of the member-parity checks


def _single(kernel, p, x, sig, r, which, v, dmu):
    """GP.fisher_information's device steps for one member: compute, fisher_terms, apply_inverse of the mean
    gradients."""
    from george_b200 import BasicSolver
    p0 = kernel.get_parameter_vector(include_frozen=True)
    kernel.set_parameter_vector(p, include_frozen=True)
    try:
        s = BasicSolver(kernel)
        s.compute(x, sig)
        terms, rows, rdiag = s.fisher_terms(r, which, v)
        return terms, rows, rdiag, s.apply_inverse(np.array(dmu.T, dtype=np.float64, order="F"))
    finally:
        kernel.set_parameter_vector(p0, include_frozen=True)


def _check_members(kernel, ndim, n, nb=3):
    from george_b200 import BasicSolver
    from george_b200._spec import flatten
    spec, which = flatten(kernel), bg._which(kernel)
    params = bg._perturbed(kernel, nb, n)
    x, sig, r = bg._inputs(n, ndim, nb, n + 1)
    rng = np.random.default_rng(n + 2)
    v = rng.uniform(0.5, 1.5, (nb, NV, n))
    dmu = rng.standard_normal((nb, NM, n))
    for rr in (r, None):
        terms, rows, rdiag, kdmu, info = BasicSolver.batch_fisher_terms(spec, params, x, sig, rr, which, v, dmu)
        assert np.all(info == 0), (n, info)
        assert (terms is None) == (rr is None)
        for b in range(nb):
            st, srows, srdiag, skdmu = _single(kernel, params[b], x, sig[b], None if rr is None else r[b], which,
                                               v[b], dmu[b])
            assert np.array_equal(rows[b], srows), (n, b, np.max(np.abs(rows[b] - srows)))
            assert np.array_equal(rdiag[b], srdiag), (n, b, np.max(np.abs(rdiag[b] - srdiag)))
            assert np.array_equal(kdmu[b].T, skdmu), (n, b)
            if rr is not None:
                for got, want, what in zip(terms, st, ("alpha", "g", "diag")):
                    assert np.array_equal(got[b], want), (n, b, what)


@pytest.mark.parametrize("name", [z[0] for z in bg._zoo()])
def test_members_match_the_single_path(gpu, name):
    _, kernel, ndim = [z for z in bg._zoo() if z[0] == name][0]
    for n in bg.SIZES:
        _check_members(kernel, ndim, n)


@pytest.mark.parametrize("n", [2048, 2049])
def test_members_match_the_single_path_either_side_of_the_single_slice_product(gpu, n):
    """From n = 2049 the products of a 132-SM H100 run in one split-K slice, below it in several."""
    from george_b200 import kernels
    _check_members(1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3), 3, n, nb=2)


# ---- the GP layer ----------------------------------------------------------------------------------------------------

def _loop(gp, vecs, y, quiet=False):
    """The per-vector path batch_fisher_information stands for: F, or (grad, F) with y."""
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
    return got.shape == want.shape and np.array_equal(got, want)


def _check_gp(gp, y, vecs, quiet=False):
    """With and without y: batch == loop bit for bit, the GP left as it was; returns the batch's (grad, F)."""
    got = []
    for yy in (None, y):
        gp.log_likelihood(y)
        st = bg._state(gp)
        got.append(gp.batch_fisher_information(vecs, yy, quiet=quiet))
        bg._assert_state(gp, st)
        assert _same(got[-1], _loop(gp, vecs, yy, quiet)), yy is None
    assert np.array_equal(got[0], got[1][1])
    gp.log_likelihood(y)
    return got[1]


def _psd_symmetric(F):
    for Fb in F:
        assert np.array_equal(Fb, Fb.T)
        w = np.linalg.eigvalsh(Fb)
        assert w[0] >= -tf.PSD_TOL * np.abs(w).max(), w


def test_co2(gpu):
    gp, _, _, y = tf._case("co2")
    rng = np.random.default_rng(5)
    vecs = gp.get_parameter_vector() + 1e-3 * rng.standard_normal((6, len(gp)))
    grad, F = _check_gp(gp, y, vecs)
    assert np.all(np.isfinite(grad)) and np.all(np.isfinite(F))
    _psd_symmetric(F)


def test_fitted_mean_with_frozen_parameters(gpu):
    gp, _, _, y = tf._case("sqexp_line_loglinear")
    for name in ("mean:b", "white_noise:s", "kernel:k1:log_constant"):
        gp.freeze_parameter(name)
    rng = np.random.default_rng(6)
    vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((5, len(gp)))
    grad, F = _check_gp(gp, y, vecs)
    assert F.shape == (5, 3, 3) and grad.shape == (5, 3)
    assert np.all(F[:, 0, 0] > 0)  # the mean block
    _psd_symmetric(F)


def test_non_constant_white_noise(gpu):
    gp, _, _, y = tf._case("sqexp_line_loglinear")
    rng = np.random.default_rng(7)
    vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((5, len(gp)))
    _, F = _check_gp(gp, y, vecs)
    _psd_symmetric(F)


def test_against_the_longdouble_brute_force(gpu, record_property):
    errs = {}
    for name in tf.WELL_CONDITIONED:
        gp, x, yerr, _ = tf._case(name)
        rng = np.random.default_rng(21)
        vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((3, len(gp)))
        F = gp.batch_fisher_information(vecs)
        _psd_symmetric(F)
        p0 = gp.get_parameter_vector()
        err = 0.0
        try:
            for b, v in enumerate(vecs):
                gp.set_parameter_vector(v)
                err = max(err, tf._rel(F[b], tf._brute(gp, x, yerr)))
        finally:
            gp.set_parameter_vector(p0)
        errs[name] = err
    record_property("batch_fisher_rel_err", errs)
    assert max(errs.values()) < tf.BRUTE_TOL, errs


def _check_failures(gp, y, vecs, bad, exc_type):
    """quiet: the loop's results, the bad members all zeros; otherwise the loop's first exception."""
    got = _check_gp(gp, y, vecs, quiet=True)
    assert np.all(got[1][bad] == 0.0) and np.all(got[0][bad] == 0.0)
    assert np.all(np.delete(got[1], bad, axis=0).any(axis=(1, 2)))
    gp.log_likelihood(y)
    st = bg._state(gp)
    with pytest.raises(exc_type) as batch_exc:
        gp.batch_fisher_information(vecs, y)
    bg._assert_state(gp, st)
    with pytest.raises(exc_type) as loop_exc:
        _loop(gp, vecs, y)
    assert str(batch_exc.value) == str(loop_exc.value)


def test_not_positive_definite_members(gpu):
    gp, y = bg._dot_gp()  # no kernel parameters: white-noise rows only
    vecs = np.full((8, len(gp)), np.log(0.1))
    bad = [2, 5]
    vecs[bad, 0] = -80.0  # K = x x^T + 1.8e-35 I: rank one, not positive definite
    _check_failures(gp, y, vecs, bad, LinAlgError)


def test_non_finite_mean_member(gpu):
    """A NaN constant mean fails the residual with y; without y the single call never evaluates the mean, so only
    the y route fails."""
    gp, y = bg._co2_gp(n=120)
    rng = np.random.default_rng(8)
    vecs = gp.get_parameter_vector() + 1e-4 * rng.standard_normal((6, len(gp)))
    vecs[3, 0] = np.nan
    got = gp.batch_fisher_information(vecs, y, quiet=True)
    assert _same(got, _loop(gp, vecs, y, quiet=True))
    assert np.all(got[0][3] == 0.0) and np.all(got[1][3] == 0.0)
    assert np.all(np.delete(got[1], 3, axis=0).any(axis=(1, 2)))
    with pytest.raises(ValueError) as batch_exc:
        gp.batch_fisher_information(vecs, y)
    with pytest.raises(ValueError) as loop_exc:
        _loop(gp, vecs, y)
    assert str(batch_exc.value) == str(loop_exc.value)
    assert _same(gp.batch_fisher_information(vecs), _loop(gp, vecs, None))


# ---- position, chunking, launches, a large batch ----------------------------------------------------------------------

def _terms(spec, params, x, sig, r, which, v, dmu):
    from george_b200 import BasicSolver
    terms, rows, rdiag, kdmu, _ = BasicSolver.batch_fisher_terms(spec, params, x, sig, r, which, v, dmu)
    return (() if terms is None else terms) + (rows, rdiag, kdmu)


def test_results_do_not_depend_on_batch_position_or_chunking(gpu, monkeypatch):
    from george_b200 import kernels
    from george_b200._spec import flatten
    kernel = 1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3)
    spec, which = flatten(kernel), bg._which(kernel)
    n, nb = 130, 12
    params = bg._perturbed(kernel, nb, 11)
    x, sig, r = bg._inputs(n, 3, nb, 12)
    rng = np.random.default_rng(13)
    v, dmu = rng.uniform(0.5, 1.5, (nb, 1, n)), rng.standard_normal((nb, 3, n))
    monkeypatch.delenv("BGP_BATCH_CHUNK", raising=False)
    for rr in (None, r):
        def call(idx):
            return _terms(spec, params[idx], x, sig[idx], None if rr is None else rr[idx], which, v[idx], dmu[idx])
        ref = call(slice(None))

        def same(got, idx_got, idx_ref):
            return all(np.array_equal(a[idx_got], b[idx_ref]) for a, b in zip(got, ref))

        assert same(call(slice(None)), slice(None), slice(None))
        for b in (0, 5, 11):
            assert same(call(slice(b, b + 1)), 0, b), b
        order = [i for i in range(nb) if i != 5] + [5]
        assert same(call(order), -1, 5)
        for chunk in ("1", "5", "64"):  # 5: two chunks of five and a ragged tail of two
            monkeypatch.setenv("BGP_BATCH_CHUNK", chunk)
            got = call(slice(None))
            monkeypatch.delenv("BGP_BATCH_CHUNK")
            assert same(got, slice(None), slice(None)), chunk


def test_launch_count_does_not_grow_with_the_batch(gpu, monkeypatch):
    from george_b200 import BasicSolver, _lib, kernels
    from george_b200._spec import flatten
    monkeypatch.delenv("BGP_BATCH_CHUNK", raising=False)
    lib = _lib.load()
    kernel = 1.3 * kernels.Matern52Kernel([0.5, 1.0, 2.0], ndim=3)
    spec, which = flatten(kernel), bg._which(kernel)
    n = 512
    params = bg._perturbed(kernel, 48, 13)
    x, sig, r = bg._inputs(n, 3, 48, 14)
    rng = np.random.default_rng(15)
    v, dmu = rng.uniform(0.5, 1.5, (48, 1, n)), rng.standard_normal((48, 2, n))
    for rr in (None, r):
        counts = []
        for nb in (1, 48):
            c0 = lib.bgp_launch_count()
            BasicSolver.batch_fisher_terms(spec, params[:nb], x, sig[:nb], None if rr is None else rr[:nb], which,
                                           v[:nb], dmu[:nb])
            counts.append(lib.bgp_launch_count() - c0)
        assert counts[0] == counts[1] > 0, (rr is None, counts)


def test_large_batch(gpu):
    import george_b200 as george
    from george_b200 import kernels
    rng = np.random.default_rng(16)
    n = 4096
    x = np.sort(rng.uniform(0, 100, n))
    y = np.sin(x) + 0.1 * rng.standard_normal(n)
    gp = george.GP(1.3 * kernels.Matern32Kernel(4.0), mean=0.1, fit_mean=True, white_noise=np.log(0.05),
                   fit_white_noise=True)
    gp.compute(x, 0.3)
    vecs = gp.get_parameter_vector() + 0.05 * rng.standard_normal((16, len(gp)))
    grad, F = gp.batch_fisher_information(vecs, y)
    assert np.all(np.isfinite(grad)) and np.all(np.isfinite(F))
    pick = [0, 7, 8, 15]
    want = _loop(gp, vecs[pick], y)
    assert np.array_equal(grad[pick], want[0]) and np.array_equal(F[pick], want[1])
    _psd_symmetric(F[pick])
