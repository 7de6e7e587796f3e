# -*- coding: utf-8 -*-
"""``tests/ou_reference.py`` against the O(n^3) longdouble references of ``tests/hiprec.py`` on the oracle's K.

The closed forms are what the large-index GPU tests (``test_gpu_zz_large_index.py``) compare the solvers with at sizes
where no O(n^3) reference runs, so each quantity they use is pinned here at n <= 500: the factor's columns, log det,
solves, the tridiagonal K^-1, ``z L^T``, ``D a``, the gradient terms (against ``einsum`` over the oracle's gradient
tensor, which also fixes the factor 1/2 and the sign of the ``log m`` derivative), the predictive mean and variance,
the leave-one-out terms of ``test_gpu_zz_loo_closed_form.py`` (``K a``, alpha, d, beta, diag(A), g and its scale
against the brute-force formula, the value and LOO predictive against refits without the point), and the Fisher
information and input gradient of ``test_gpu_zz_fisher_grad_x_closed_form.py`` (F against the trace formula over the
oracle's gradient tensor; dx and its scale against the contraction with the oracle's x-gradient, and against central
differences of the log-likelihood, which do not go through that contraction).
The differences are the float64 rounding of K's entries carried through cond(K) <= 10 (largest measured: 1.5e-15, in
the LOO diag(A); bar 1e-14); the central differences have their own bar.
"""
import numpy as np
import pytest

import hiprec
import ou_reference

LD = np.longdouble
TOL = 1e-14

# (n, c, m, gap): gaps are uniform(gap) * sqrt(m); the last case spans ~1100 length scales, so the far entries of the
# float64 K underflow to 0 while the closed form keeps them (exp(-1100) ~ 1e-478 in longdouble)
CASES = [(1, 1.0, 1.0, (0.2, 1.0)), (2, 0.7, 2.0, (0.2, 1.0)), (65, 1.0, 1.0, (0.2, 1.0)),
         (300, 2.5, 0.04, (0.2, 1.0)), (500, 0.3, 9.0, (0.2, 1.0)), (500, 1.7, 0.5, (1.5, 3.0))]


def _case(n, c, m, gap):
    from george_b200 import kernels
    from george_b200._spec import flatten
    import oracle
    x = ou_reference.exp_problem(n, np.sqrt(m), seed=n, x0=-0.3 * n * np.sqrt(m), gap=gap)
    kernel = c * kernels.ExpKernel(m)
    spec = flatten(kernel)
    K = oracle.value_symmetric(spec, x[:, None])
    return x, kernel, spec, K, ou_reference.OU(x, c, m)


def _rel(A, Ref):
    Ref = np.asarray(Ref, dtype=LD)
    den = np.max(np.abs(Ref))
    return float(np.max(np.abs(np.asarray(A, dtype=LD) - Ref)) / (den if den > 0 else 1))


@pytest.mark.parametrize("n,c,m,gap", CASES)
def test_closed_forms_match_the_longdouble_factorisation(oracle, n, c, m, gap):
    x, kernel, spec, K, ou = _case(n, c, m, gap)
    if gap[0] > 1:
        assert np.sum(K == 0) > n * n // 10  # the case it is meant to be (12 % of the entries)
    L = hiprec.chol_ld(K)
    assert abs(float(ou.logdet() - hiprec.logdet_ld(L))) <= TOL * max(1.0, abs(float(hiprec.logdet_ld(L))))
    assert _rel(ou.chol_columns(np.arange(n)), L) <= TOL
    cols = sorted({0, n // 2, n - 1})
    assert np.array_equal(ou.chol_columns(cols), ou.chol_columns(np.arange(n))[:, cols])

    rng = np.random.default_rng(n + 1)
    B = rng.standard_normal((n, 3))
    X = hiprec.solve_ld(L, B)
    assert _rel(ou.solve(B), X) <= TOL
    assert _rel(ou.solve(B[:, 0]), X[:, 0]) <= TOL
    assert _rel(ou.inv_chol(B), _lower_solve(L, B)) <= TOL

    Kinv = hiprec.solve_ld(L, np.eye(n))
    d, e = ou.inv_tridiag()
    T = np.diag(d)
    if n > 1:
        T += np.diag(e, 1) + np.diag(e, -1)
    assert _rel(T, Kinv) <= TOL

    Z = rng.standard_normal((4, n))
    assert _rel(ou.sqrt_rows(Z), Z.astype(LD) @ L.T) <= TOL
    assert _rel(ou.sqrt_rows(Z[0]), Z[0].astype(LD) @ L.T) <= TOL


def _lower_solve(L, B):
    X = np.array(B, dtype=LD)
    for i in range(L.shape[0]):
        X[i] = (X[i] - L[i, :i] @ X[:i]) / L[i, i]
    return X


@pytest.mark.parametrize("n,c,m,gap", CASES)
def test_gradient_terms_match_the_oracle_gradient_tensor(oracle, n, c, m, gap):
    x, kernel, spec, K, ou = _case(n, c, m, gap)
    assert list(kernel.get_parameter_names(include_frozen=True)) == ["k1:log_constant", "k2:metric:log_M_0_0"]
    L = hiprec.chol_ld(K)
    Kinv = hiprec.solve_ld(L, np.eye(n))
    dK = oracle.gradient_general(spec, [1, 1], x[:, None], x[:, None]).astype(LD)
    # D = 2 dK/dlog m
    a = np.random.default_rng(n + 2).standard_normal(n)
    assert _rel(ou.apply_d(a), 2 * dK[:, :, 1] @ a.astype(LD)) <= TOL
    assert abs(float(ou.trace_kinv_d() - 2 * np.sum(Kinv * dK[:, :, 1]))) <= TOL * max(1.0, float(np.sum(np.abs(Kinv * dK[:, :, 1]))))

    r = np.sin(x / np.sqrt(m)) + 0.5
    alpha_ref = Kinv @ r.astype(LD)
    A = np.outer(alpha_ref, alpha_ref) - Kinv
    g_ref = np.einsum("ijk,ij->k", dK, A)
    scale = np.einsum("ijk,ij->k", np.abs(dK), np.abs(A))
    alpha, g, diag = ou.grad_terms(r)
    assert _rel(alpha, alpha_ref) <= TOL
    assert np.all(np.abs(g - g_ref) <= TOL * scale), (g, g_ref, scale)
    assert _rel(diag, np.diag(A)) <= TOL


@pytest.mark.parametrize("n,c,m,gap", CASES)
def test_loo_terms_match_the_longdouble_formula(oracle, n, c, m, gap):
    """``loo_terms`` against the brute-force formula on the oracle's K (``_ld_formula`` of test_gpu_loo.py), g against
    ``einsum`` over the oracle's gradient tensor, and the value and predictive against N - 1-point refits."""
    x, kernel, spec, K, ou = _case(n, c, m, gap)
    L = hiprec.chol_ld(K)
    Kinv = hiprec.solve_ld(L, np.eye(n))
    Kinv = (Kinv + Kinv.T) / 2
    dK = oracle.gradient_general(spec, [1, 1], x[:, None], x[:, None]).astype(LD)
    a = np.random.default_rng(n + 4).standard_normal(n)
    assert _rel(ou.apply_k(a), K.astype(LD) @ a.astype(LD)) <= TOL
    assert _rel(ou.apply_k(a), dK[:, :, 0] @ a.astype(LD)) <= TOL  # dK/dlog c = K

    r = np.sin(x / np.sqrt(m)) + 0.1 * np.random.default_rng(n + 5).standard_normal(n)
    alpha_ref = Kinv @ r.astype(LD)
    d_ref = np.diag(Kinv).copy()
    q = alpha_ref / d_ref
    beta_ref = Kinv @ q
    w = (1 + alpha_ref * q) / (2 * d_ref)
    A = (np.outer(beta_ref, alpha_ref) + np.outer(alpha_ref, beta_ref)) / 2 - Kinv @ (w[:, None] * Kinv)
    g_ref = np.einsum("ijk,ij->k", dK, A)
    scale = np.einsum("ijk,ij->k", np.abs(dK), np.abs(A))
    value_ref = np.sum(-np.log(2 * LD(np.pi)) / 2 + np.log(d_ref) / 2 - alpha_ref ** 2 / (2 * d_ref))

    t = ou.loo_terms(r)
    assert _rel(t["alpha"], alpha_ref) <= TOL
    assert _rel(t["d"], d_ref) <= TOL
    assert _rel(t["beta"], beta_ref) <= TOL
    assert _rel(t["diagA"], np.diag(A)) <= TOL
    assert np.all(np.abs(t["g"] - g_ref) <= TOL * scale), (t["g"], g_ref, scale)
    assert np.all(t["gscale"] >= scale * (1 - TOL)), (t["gscale"], scale)  # an upper bound
    assert np.all(t["gscale"] <= 4 * scale), (t["gscale"], scale)          # and not a loose one
    assert abs(float(t["value"] - value_ref)) <= TOL * float(np.sum(np.abs(np.log(d_ref)) + alpha_ref ** 2 / d_ref) + n)

    # the LOO predictive and each point's term of the value against refits without the point
    for i in sorted({0, n // 2, n - 1}):
        k = np.delete(np.arange(n), i)
        if k.size:
            Li = hiprec.chol_ld(K[np.ix_(k, k)])
            mu = K[i, k].astype(LD) @ hiprec.solve_ld(Li, r[k].astype(LD))
            var = LD(K[i, i]) - K[i, k].astype(LD) @ hiprec.solve_ld(Li, K[k, i].astype(LD))
        else:
            mu, var = LD(0), LD(K[i, i])
        assert abs(float(r[i] - t["alpha"][i] / t["d"][i] - mu)) <= TOL * max(1.0, float(np.max(np.abs(r))))
        assert abs(float(1 / t["d"][i] - var)) <= TOL * c
        term = -np.log(2 * LD(np.pi) * var) / 2 - (r[i] - mu) ** 2 / (2 * var)
        own = -np.log(2 * LD(np.pi)) / 2 + np.log(t["d"][i]) / 2 - t["alpha"][i] ** 2 / (2 * t["d"][i])
        assert abs(float(own - term)) <= TOL * max(1.0, abs(float(term)))


@pytest.mark.parametrize("n,c,m,gap", CASES)
def test_fisher_matches_the_longdouble_trace(oracle, n, c, m, gap):
    """``fisher`` against ``1/2 tr(K^-1 dK_p K^-1 dK_q)`` over the oracle's gradient tensor and ``1^T K^-1 1``, and
    ``factor_terms`` against the log-likelihood of the longdouble factorisation."""
    x, kernel, spec, K, ou = _case(n, c, m, gap)
    L = hiprec.chol_ld(K)
    Kinv = hiprec.solve_ld(L, np.eye(n))
    dK = oracle.gradient_general(spec, [1, 1], x[:, None], x[:, None]).astype(LD)
    KdK = [Kinv @ dK[:, :, p] for p in range(2)]
    F_ref = np.zeros((3, 3), dtype=LD)
    F_ref[0, 0] = np.sum(Kinv)
    scale = np.zeros((3, 3), dtype=LD)
    scale[0, 0] = np.sum(np.abs(Kinv))
    for p in range(2):
        for q in range(2):
            F_ref[1 + p, 1 + q] = np.sum(KdK[p] * KdK[q].T) / 2
            scale[1 + p, 1 + q] = np.sum(np.abs(KdK[p]) * np.abs(KdK[q].T)) / 2
    F = ou.fisher()
    assert np.all(np.abs(F - F_ref) <= TOL * scale), (F, F_ref)
    assert np.all(F[0, 1:] == 0) and np.all(F[1:, 0] == 0)
    assert np.array_equal(ou.fisher(mean=False), F[1:, 1:])
    assert F[1, 1] == LD(n) / 2
    assert abs(float(F[1, 2] - ou.trace_kinv_d() / 4)) <= TOL * float(scale[1, 2])

    r = np.sin(x / np.sqrt(m)) + 0.5
    ll_ref = -(r.astype(LD) @ hiprec.solve_ld(L, r.astype(LD)) + hiprec.logdet_ld(L) + n * np.log(2 * LD(np.pi))) / 2
    ll = np.sum(ou.factor_terms(r))
    assert abs(float(ll - ll_ref)) <= TOL * float(np.sum(np.abs(ou.factor_terms(r))))


# Central differences in the scaled gaps, extrapolated twice (truncation O(h^6)): the rounding of the factor terms over
# the step, ~1e-19 / FD_STEP, limits them (largest measured: 4.2e-14, the widely spaced case, where scale is smallest)
FD_STEP = 1e-3
FD_TOL = 5e-13


@pytest.mark.parametrize("n,c,m,gap", CASES)
def test_grad_x_matches_the_contraction_and_differences(oracle, n, c, m, gap):
    """``grad_x`` against ``sum_j (alpha alpha^T - K^-1)_ij dk_ij/dx_i`` with the oracle's x-gradient and the
    longdouble K^-1, and against central differences of the log-likelihood in each x_i (through ``factor_terms``,
    whose sum is pinned to the factorisation's log-likelihood above); its scale bounds the contraction's terms."""
    x, kernel, spec, K, ou = _case(n, c, m, gap)
    L = hiprec.chol_ld(K)
    Kinv = hiprec.solve_ld(L, np.eye(n))
    Kinv = (Kinv + Kinv.T) / 2
    dkdx = oracle.x_gradient_general(spec, 1, x[:, None], x[:, None])[:, :, 0].astype(LD)
    r = np.sin(x / np.sqrt(m)) + 0.1 * np.random.default_rng(n + 6).standard_normal(n)
    alpha = Kinv @ r.astype(LD)
    A = np.outer(alpha, alpha) - Kinv
    dx_ref = np.sum(A * dkdx, axis=1)
    bound = np.sum(np.abs(A) * np.abs(dkdx), axis=1)
    dx, scale = ou.grad_x(r)
    assert np.all(np.abs(dx - dx_ref) <= TOL * scale), float(np.max(np.abs(dx - dx_ref) / scale))
    assert np.all(scale >= bound * (1 - TOL)), (scale, bound)
    assert np.sum(scale) <= 4 * np.sum(bound), (np.sum(scale), np.sum(bound))
    assert abs(float(np.sum(dx))) <= TOL * float(np.sum(scale))

    # d t_j / d gap_j per factor, then dx_i = G_i - G_{i+1}
    def diff(h):
        eta = LD(h)  # a step of h length scales in every gap
        return (ou.factor_terms(r, ou.delta + eta) - ou.factor_terms(r, ou.delta - eta)) / (2 * h * ou.ell)

    def richardson(h):
        return (4 * diff(h / 2) - diff(h)) / 3
    G = (16 * richardson(FD_STEP / 2) - richardson(FD_STEP)) / 15
    G[0] = 0
    dx_fd = G.copy()
    dx_fd[:-1] -= G[1:]
    assert np.all(np.abs(dx - dx_fd) <= FD_TOL * scale), float(np.max(np.abs(dx - dx_fd) / scale))


@pytest.mark.parametrize("n,c,m,gap", CASES)
def test_prediction_matches_the_dense_formulas(oracle, n, c, m, gap):
    x, kernel, spec, K, ou = _case(n, c, m, gap)
    L = hiprec.chol_ld(K)
    ell = np.sqrt(m)
    rng = np.random.default_rng(n + 3)
    # inside the data, on a data point, and beyond either end
    t = np.concatenate((rng.uniform(x[0], x[-1], 16), [x[n // 2], x[0] - 0.7 * ell, x[-1] + 2.0 * ell]))
    y = rng.standard_normal(n)
    alpha = hiprec.solve_ld(L, y)
    Kts = oracle.value_general(spec, t[:, None], x[:, None]).astype(LD)
    W = _lower_solve(L, Kts.T)
    mean, var = ou.predict(t, ou.solve(y))
    assert _rel(mean, Kts @ alpha) <= TOL
    assert np.max(np.abs(var - (LD(c) - np.sum(W * W, axis=0)))) <= TOL * c
    assert abs(float(var[16])) <= TOL * c  # no variance left at a data point
