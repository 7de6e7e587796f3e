# -*- coding: utf-8 -*-
"""``tests/matern_reference.py`` against the O(n^3) longdouble references of ``tests/hiprec.py`` on the oracle's K.

The state-space reference is what ``test_gpu_zz_matern_state_space.py`` compares the solvers with at N = 2^18, where
no O(n^3) reference runs, so every output it uses is pinned here at n <= 600: log det, y^T K^-1 y, K^-1 Y, diag(K^-1),
the predictive mean and variance, the leave-one-out terms (against refits without the point) and the log-likelihood
gradient (against ``0.5 tr((alpha alpha^T - K^-1) dK)`` over the oracle's gradient tensor).  The points are clustered,
with gaps from 1e-6 to 50 length scales, and yerr varies from point to point.

The dense side factors the float64 K, whose entries are rounded by 1.1e-16; the state space works from the exact
kernel.  Their difference is that rounding carried through cond(K) (up to 1.2e4 here), so the bars are stated relative
to the size of each result; largest measured 6.2e-14 (diag(K^-1) of Matern-5/2 at n = 600), bar 3e-13.
"""
import numpy as np
import pytest

import hiprec
import matern_reference as mr

LD = np.longdouble
TOL = 3e-13

# (name, terms): a one-term kernel is c * kernel(m) as (kind, c, m); sums are block-diagonal states
KERNELS = [
    ("m32", [("m32", 1.3, 0.7)]),
    ("m52", [("m52", 0.8, 2.0)]),
    ("m32+exp", [("m32", 1.0, 1.0), ("exp", 0.4, 9.0)]),
    ("m52+exp", [("m52", 2.0, 0.5), ("exp", 0.3, 4.0)]),
]


def _kernel(terms):
    from george_b200 import kernels
    cls = {"m32": kernels.Matern32Kernel, "m52": kernels.Matern52Kernel, "exp": kernels.ExpKernel}
    out = None
    for kind, c, m in terms:
        k = c * cls[kind](m)
        out = k if out is None else out + k
    return out


def _points(n, ell, seed):
    """Clusters of points 1e-3 to 0.3 length scales apart, separated by gaps of 2 to 50 length scales, with a pair
    1e-6 length scales apart in each cluster and yerr from 0.02 to 0.5."""
    rng = np.random.default_rng(seed)
    gaps = rng.uniform(1e-3, 0.3, n) * ell
    gaps[rng.choice(n, n // 40, replace=False)] = rng.uniform(2.0, 50.0, n // 40) * ell
    gaps[rng.choice(n, n // 60, replace=False)] = 1e-6 * ell
    x = np.cumsum(gaps) - 3.0
    return x, rng.uniform(0.02, 0.5, n)


def _case(oracle, terms, n, seed):
    from george_b200._spec import flatten
    ell = min(np.sqrt(m) for _, _, m in terms)
    x, sigma = _points(n, ell, seed)
    spec = flatten(_kernel(terms))
    K = oracle.value_symmetric(spec, x[:, None])
    K[np.diag_indices(n)] += sigma * sigma
    return x, sigma, spec, K, mr.StateSpace(x, sigma, terms)


def _rel(A, Ref):
    Ref = np.asarray(Ref, dtype=LD)
    return float(np.max(np.abs(np.asarray(A, dtype=LD) - Ref)) / np.max(np.abs(Ref)))


@pytest.mark.parametrize("kind", ["exp", "m32", "m52"])
def test_transition_and_stationary_covariance(kind):
    """Pinf solves the Lyapunov equation; h^T A(D) Pinf h is the covariance function; Q keeps the semigroup identity
    Q(2D) = A(D) Q(D) A(D)^T + Q(D) and its leading term q D at gaps down to 1e-6 length scales."""
    t = mr.Term(kind, 1.7, 0.8)
    L = t.F @ t.Pinf + t.Pinf @ t.F.T
    q = -L[-1, -1]
    L[-1, -1] = 0
    assert q > 0 and np.max(np.abs(L)) <= 1e-18 * q
    scale = 1 / t.lam
    gaps = np.array([1e-6, 1e-4, 0.01, 0.3, 1.0, 7.0, 40.0], dtype=LD) * scale
    A = t.transition(gaps)
    assert _rel(A[:, 0, :] @ t.Pinf[:, 0], t.value(gaps)) <= 1e-18
    ss = mr.StateSpace(np.zeros(1), 1.0, [(kind, 1.7, 0.8)])
    for D in gaps:
        A1, Q1 = [v[1] for v in ss._steps(np.array([0.0, D], dtype=LD))]
        A2, Q2 = [v[1] for v in ss._steps(np.array([0.0, 2 * D], dtype=LD))]
        assert np.max(np.abs(A1 @ A1 - A2)) <= 1e-17 * np.max(np.abs(A1)) ** 2
        assert np.max(np.abs(A1 @ Q1 @ A1.T + Q1 - Q2)) <= 1e-18 * np.max(np.abs(t.Pinf))
        if D < 1e-3 * scale:  # Q ~ q D e_p e_p^T to first order
            assert abs(Q1[-1, -1] / (q * D) - 1) <= 10 * t.lam * D


@pytest.mark.parametrize("name,terms", KERNELS)
@pytest.mark.parametrize("n", [1, 2, 240, 600])
def test_solves_and_prediction_match_the_longdouble_factorisation(oracle, name, terms, n):
    x, sigma, spec, K, ss = _case(oracle, terms, n, seed=n)
    if n > 2:
        assert np.any(np.diff(x) < 1e-5) and np.any(np.diff(x) > 2.0)
    L = hiprec.chol_ld(K)
    rng = np.random.default_rng(n + 1)
    Y = rng.standard_normal((n, 3))
    t = np.concatenate([rng.uniform(x[0] - 1, x[-1] + 1, 12), x[[0, n // 2, n - 1]]])
    res = ss.run(Y, t)
    ld_ref = hiprec.logdet_ld(L)
    assert abs(float(res["logdet"] - ld_ref)) <= TOL * max(1.0, float(np.sum(np.abs(np.log(np.diag(L))))))
    X = hiprec.solve_ld(L, Y)
    assert _rel(res["alpha"], X) <= TOL
    assert _rel(res["quad"], np.sum(Y * X, axis=0)) <= TOL
    assert _rel(ss.run(Y[:, 0])["alpha"], X[:, 0]) <= TOL
    Kinv = hiprec.solve_ld(L, np.eye(n))
    assert _rel(res["d"], np.diag(Kinv)) <= TOL
    Kts = oracle.value_general(spec, t[:, None], x[:, None]).astype(LD)
    kss = oracle.value_diagonal(spec, t[:, None], t[:, None]).astype(LD)
    assert _rel(res["mean"], Kts @ X) <= TOL
    var_ref = kss - np.sum(Kts * (Kts @ Kinv), axis=1)
    assert np.max(np.abs(res["var"] - var_ref)) <= TOL * np.max(kss)


@pytest.mark.parametrize("name,terms", KERNELS)
def test_loo_matches_refits_without_the_point(oracle, name, terms):
    """The LOO mean, variance and each point's term of the value at the ends, both points of the closest pair and a
    spread of others; the value as the sum of the terms."""
    n = 240
    x, sigma, spec, K, ss = _case(oracle, terms, n, seed=7)
    y = np.sin(x) + 0.3 * np.random.default_rng(8).standard_normal(n)
    res = ss.run(y)
    loo = ss.loo(y, res)
    close = int(np.argmin(np.diff(x)))
    a, d = res["alpha"], res["d"]
    terms_ref = -np.log(2 * LD(np.pi)) / 2 + np.log(d) / 2 - a * a / (2 * d)
    assert abs(float(loo["value"] - np.sum(terms_ref))) <= 1e-17 * float(np.sum(np.abs(terms_ref)))
    for i in sorted({0, n - 1, close, close + 1} | set(range(5, n, 23))):
        k = np.delete(np.arange(n), i)
        Li = hiprec.chol_ld(K[np.ix_(k, k)])
        w = hiprec.solve_ld(Li, K[k, i].astype(LD))
        mu = w @ y[k].astype(LD)
        var = LD(K[i, i]) - K[i, k].astype(LD) @ w
        assert abs(float(loo["mean"][i] - mu)) <= TOL * max(1.0, float(np.max(np.abs(y))))
        assert abs(float(loo["var"][i] - var)) <= TOL * float(K[i, i])
        term = -np.log(2 * LD(np.pi) * var) / 2 - (y[i] - mu) ** 2 / (2 * var)
        assert abs(float(terms_ref[i] - term)) <= TOL * max(1.0, abs(float(term)))


@pytest.mark.parametrize("name,terms", KERNELS)
def test_gradient_matches_the_oracle_gradient_tensor(oracle, name, terms):
    """Every kernel parameter by finite differences; log c of one-term kernels also from the smoother."""
    n = 240
    x, sigma, spec, K, ss = _case(oracle, terms, n, seed=11)
    y = np.sin(x) + 0.3 * np.random.default_rng(12).standard_normal(n)
    P = 2 * len(terms)
    dK = oracle.gradient_general(spec, np.ones(P), x[:, None], x[:, None]).astype(LD)
    L = hiprec.chol_ld(K)
    Kinv = hiprec.solve_ld(L, np.eye(n))
    alpha = Kinv @ y.astype(LD)
    A = np.outer(alpha, alpha) - Kinv
    g_ref = np.einsum("ijk,ij->k", dK, A) / 2
    scale = np.einsum("ijk,ij->k", np.abs(dK), np.abs(A)) / 2
    theta = np.log(np.array([v for _, c, m in terms for v in (c, m)], dtype=LD))

    def member(th):
        return sigma, [(kind, np.exp(th[2 * q]), np.exp(th[2 * q + 1])) for q, (kind, _, _) in enumerate(terms)]

    g_fd = np.array([mr.grad_fd(member, theta, x, y, p) for p in range(P)])
    assert np.all(np.abs(g_fd - g_ref) <= TOL * scale), (g_fd, g_ref, scale)
    if len(terms) == 1:
        g_c = ss.grad_log_c(y, ss.run(y))
        assert abs(g_c - g_ref[0]) <= TOL * scale[0]
        assert abs(g_c - g_fd[0]) <= 1e-15 * scale[0]  # the two longdouble routes


def test_batched_members_match_single_runs():
    """``log_likelihoods`` runs its members in one loop: each equals its own ``StateSpace``."""
    x, sigma = _points(300, 1.0, seed=3)
    y = np.cos(x)
    members = [(sigma, [("m32", 1.0, 1.0)]), (0.5 * sigma, [("m32", 2.0, 0.3)]), (sigma, [("m32", 0.1, 5.0)])]
    ll = mr.log_likelihoods(x, members, y)
    for b, (s, terms) in enumerate(members):
        assert ll[b] == mr.StateSpace(x, s, terms).log_likelihood(y)
