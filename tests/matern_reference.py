# -*- coding: utf-8 -*-
"""Exact O(n) references for Matern-3/2, Matern-5/2 and their sums with ``ExpKernel`` on sorted 1-D inputs with noise
(test infrastructure; numpy only).

On a line, ``c * Matern32Kernel(m)``, ``c * Matern52Kernel(m)`` and ``c * ExpKernel(m)`` are the covariances of
stationary Markov processes with p = 2, 3 and 1 state dimensions (Hartikainen & Sarkka, "Kalman filtering and
smoothing solutions to temporal Gaussian process regression models", 2010).  With george's ``r^2 = d^2 / m``:

    Matern-3/2: k(d) = c (1 + lam d) exp(-lam d),                 lam = sqrt(3 / m)
    Matern-5/2: k(d) = c (1 + lam d + lam^2 d^2 / 3) exp(-lam d),  lam = sqrt(5 / m)
    Exp:        k(d) = c exp(-lam d),                              lam = 1 / sqrt(m)

The state is (f, f', ..., f^(p-1)) with the companion matrix F of (s + lam)^p, so ``N = F + lam I`` is nilpotent and
the transition over a gap ``D`` is exactly ``A(D) = exp(F D) = exp(-lam D) sum_{k<p} N^k D^k / k!``.  The stationary
covariance ``Pinf`` (``Pinf_ij = (-1)^j k^(i+j)(0)``) solves ``F Pinf + Pinf F^T + q e_p e_p^T = 0``, and the process
noise of a step is ``Q = Pinf - A Pinf A^T``.  A sum of kernels is the block-diagonal state of its terms, observed
through ``h``, which is 1 at the first state of every block.

With ``K_y = K + diag(sigma^2)`` (sigma > 0), one forward Kalman filter gives the innovations ``v_i`` and their
variances ``S_i``, so that ``K_y = B^-1 diag(S) B^-T`` with B unit lower triangular (``v = B y``):

* ``log det K_y = sum_i log S_i`` and ``y^T K_y^-1 y = sum_i v_i^2 / S_i``;
* ``K_y^-1 Y = B^T diag(1 / S) B Y``: the adjoint of the filter, a backward sweep over the same gains G
  (``u_i = w_i - G_i . rho^_i``, ``rho_i = rho^_i + h u_i``, ``rho^_(i-1) = A_i^T rho_i``, ``w = v / S``);
* ``diag(K_y^-1)_i = 1 / S_i + G_i^T Psi_i G_i``, with ``Omega_i = h h^T / S_i + (I - G_i h^T)^T Psi_i (I - G_i h^T)``
  and ``Psi_(i-1) = A_i^T Omega_i A_i``: a sum of non-negative terms, nothing cancels;
* at a test point t merged into the sweep with no measurement, ``E[s_t | y] = m^-_t + P^-_t rho^_t`` and
  ``Var(s_t | y) = P^-_t - P^-_t Psi_t P^-_t``, so the predictive mean ``K(t, x) K_y^-1 y`` and variance
  ``k(t, t) - K(t, x) K_y^-1 K(x, t)`` are those of h^T s_t.

This is the Bryson-Frazier form of the Rauch-Tung-Striebel smoother: it never inverts a state covariance, so a gap of
1e-6 length scales (A ~ I, Q ~ 0) costs no accuracy.  Everything is ``np.longdouble`` (x87 80-bit on x86-64, eps
1.1e-19): ``Q`` loses at most ~lam D of its relative accuracy to cancellation, which at D = 1e-6 length scales is
still ~1e-13 of Q and far below 1e-19 of c absolutely.  The distance of a float64 result from these values is the
float64 result's own error.

For the kernel ``c * k(m)`` of one term, the log-likelihood gradient with respect to log c follows from alpha and d
(``dK / dlog c = K = K_y - diag(sigma^2)``); every other parameter's derivative is a Richardson-extrapolated central
difference of the longdouble log-likelihood (``grad_fd``).
"""
import math

import numpy as np

LD = np.longdouble
assert np.finfo(LD).nmant >= 63, (
    "np.longdouble has a {0}-bit mantissa here: the extended-precision reference needs the 80-bit x87 format"
    .format(np.finfo(LD).nmant))

ORDER = {"exp": 1, "m32": 2, "m52": 3}


class Term(object):
    """One term ``c * kernel(m)`` of a sum: ``kind`` is "exp", "m32" or "m52"."""

    def __init__(self, kind, c, m):
        self.kind, self.c, self.m = kind, LD(c), LD(m)
        self.p = p = ORDER[kind]
        self.lam = {"exp": 1 / np.sqrt(self.m), "m32": np.sqrt(3 / self.m), "m52": np.sqrt(5 / self.m)}[kind]
        lam = self.lam
        # (s + lam)^p = s^p + a_(p-1) s^(p-1) + ... + a_0
        a = [LD(math.comb(p, k)) * lam ** (p - k) for k in range(p)]
        F = np.zeros((p, p), dtype=LD)
        F[np.arange(p - 1), np.arange(1, p)] = 1
        F[p - 1, :] = [-ak for ak in a]
        self.F = F
        N = F + lam * np.eye(p, dtype=LD)
        self.Npow = [np.linalg.matrix_power(N, k) if k else np.eye(p, dtype=LD) for k in range(p)]
        c = self.c
        self.Pinf = {"exp": c * np.eye(1, dtype=LD),
                     "m32": c * np.diag([LD(1), lam ** 2]),
                     "m52": c * np.array([[1, 0, -lam ** 2 / 3], [0, lam ** 2 / 3, 0], [-lam ** 2 / 3, 0, lam ** 4]],
                                         dtype=LD)}[kind]

    def value(self, d):
        """``k(d)`` in longdouble (d >= 0)."""
        t = self.lam * np.asarray(d, dtype=LD)
        poly = {"exp": 1, "m32": 1 + t, "m52": 1 + t + t * t / 3}[self.kind]
        return self.c * poly * np.exp(-t)

    def transition(self, gaps):
        """``A(D)`` for every gap: ``(len(gaps), p, p)``."""
        gaps = np.asarray(gaps, dtype=LD)
        A = np.zeros((gaps.size, self.p, self.p), dtype=LD)
        for k, Nk in enumerate(self.Npow):
            A += (gaps ** k / math.factorial(k))[:, None, None] * Nk
        return np.exp(-self.lam * gaps)[:, None, None] * A


class StateSpace(object):
    """``K_y = sum_terms K_term + diag(sigma^2)`` at the sorted points ``x``, ``sigma`` > 0."""

    def __init__(self, x, sigma, terms):
        x = np.asarray(x, dtype=np.float64).reshape(-1)
        if x.size > 1 and not np.all(np.diff(x) >= 0):
            raise ValueError("x must be sorted")
        self.n = x.size
        self.x = x
        self.s2 = np.asarray(sigma, dtype=np.float64).astype(LD) ** 2 * np.ones(self.n, dtype=LD)
        if not np.all(self.s2 > 0):
            raise ValueError("the state-space reference needs noise at every point")
        self.terms = [Term(*t) for t in terms]
        self.p = sum(t.p for t in self.terms)
        self.h = np.zeros(self.p, dtype=LD)
        off = 0
        self.blocks = []
        for t in self.terms:
            self.h[off] = 1
            self.blocks.append(slice(off, off + t.p))
            off += t.p
        self.Pinf = np.zeros((self.p, self.p), dtype=LD)
        for t, b in zip(self.terms, self.blocks):
            self.Pinf[b, b] = t.Pinf

    def kernel(self, d):
        """The covariance at distance d (longdouble)."""
        return sum(t.value(np.abs(np.asarray(d, dtype=LD))) for t in self.terms)

    def _steps(self, z):
        """``(A, Q)`` of every step of the sorted sequence z (``A[0]``, ``Q[0]`` unused)."""
        z = np.asarray(z, dtype=LD)
        gaps = np.zeros(z.size, dtype=LD)
        gaps[1:] = np.diff(z)
        A = np.zeros((z.size, self.p, self.p), dtype=LD)
        for t, b in zip(self.terms, self.blocks):
            A[:, b, b] = t.transition(gaps)
        Q = self.Pinf - A @ self.Pinf @ np.swapaxes(A, 1, 2)
        return A, (Q + np.swapaxes(Q, 1, 2)) / 2

    def run(self, Y=None, t=None, smooth=True):
        """One forward filter and (with ``smooth``) one backward sweep.

        ``Y``: ``(n,)`` or ``(n, k)`` right-hand sides (default: none); ``t``: test points (any order).  Returns a
        dict with ``logdet``, ``quad`` (``(k,)``: ``Y_j^T K_y^-1 Y_j``) and, with ``smooth``, ``alpha`` (K_y^-1 Y, Y's
        shape), ``d`` (diag K_y^-1) and at the test points ``mean`` (``(nt, k)``: K(t, x) K_y^-1 Y) and ``var``."""
        n, p, h = self.n, self.p, self.h
        Y0 = np.zeros((n, 0)) if Y is None else np.asarray(Y, dtype=np.float64)
        t = np.zeros(0) if t is None else np.asarray(t, dtype=np.float64).reshape(-1)
        f = _forward([self], Y0.reshape(n, -1), t)
        out = dict(logdet=f["logdet"][0], quad=f["quad"][0])
        if not smooth:
            return out
        order, is_test, A, M = f["order"], f["is_test"], f["A"][:, 0], f["order"].size
        S, G, W, Zt = f["S"][0], f["G"][0], f["W"][0], f["Zt"][:, 0]
        k = W.shape[1]
        # backward: R = [Psi | rho^] (p, p + k)
        alpha = np.zeros((n, k), dtype=LD)
        d = np.zeros(n, dtype=LD)
        mean = np.zeros((t.size, k), dtype=LD)
        var = np.zeros(t.size, dtype=LD)
        R = np.zeros((p, p + k), dtype=LD)
        for j in range(M - 1, -1, -1):
            i = order[j]
            if is_test[j]:
                Pm, mm = Zt[i - n][:, :p], Zt[i - n][:, p:]
                ph = Pm @ h
                mean[i - n] = h @ mm + ph @ R[:, p:]
                var[i - n] = h @ ph - ph @ R[:, :p] @ ph
            else:
                g, s = G[i], S[i]
                b = R[:, :p] @ g
                u = W[i] - g @ R[:, p:]
                alpha[i] = u
                d[i] = 1 / s + g @ b
                # Omega = Psi - h b^T - b h^T + (1 / S + g . b) h h^T
                R[:, :p] += d[i] * np.outer(h, h) - np.outer(h, b) - np.outer(b, h)
                R[:, p:] += np.outer(h, u)
            if j:
                R = A[j].T @ R
                R[:, :p] = R[:, :p] @ A[j]
        out.update(alpha=alpha.reshape(Y0.shape), d=d, mean=mean, var=var)
        return out

    # ---- derived quantities -----------------------------------------------------------------------------------------
    def log_likelihood(self, y):
        res = self.run(y, smooth=False)
        return -(self.n * np.log(2 * LD(np.pi)) + res["logdet"] + res["quad"][0]) / 2

    def grad_log_c(self, y, res):
        """d log-likelihood / d log c of a one-term kernel from ``res = run(y)``: with ``K = K_y - diag(sigma^2)``,
        ``alpha^T K alpha = alpha . y - sum sigma^2 alpha^2`` and ``tr(K_y^-1 K) = n - sum sigma^2 d``."""
        assert len(self.terms) == 1
        a = res["alpha"].reshape(-1)
        y = np.asarray(y, dtype=np.float64).astype(LD)
        return (a @ y - np.sum(self.s2 * a * a) - self.n + np.sum(self.s2 * res["d"])) / 2

    def loo(self, y, res):
        """The leave-one-out terms from ``res = run(y)``: mean, variance and value (GPML eqs. 5.10-5.11)."""
        a = res["alpha"].reshape(-1)
        d = res["d"]
        y = np.asarray(y, dtype=np.float64).astype(LD)
        value = np.sum(-np.log(2 * LD(np.pi)) / 2 + np.log(d) / 2 - a * a / (2 * d))
        return dict(mean=y - a / d, var=1 / d, value=value)


def _forward(models, Y, t):
    """The Kalman filter of every model in ``models`` (``StateSpace`` objects on the same x, with the same kinds of
    terms) over the data and the test points ``t`` merged in order, in one loop: per model its log det and
    ``Y^T K_y^-1 Y``, and per data point S, G and w = v / S; the predicted [P | m] at each test point."""
    B, n, p, h = len(models), models[0].n, models[0].p, models[0].h
    Yk = np.asarray(Y, dtype=np.float64).astype(LD)
    k = Yk.shape[1]
    z = np.concatenate([models[0].x, t])
    order = np.argsort(z, kind="stable")  # a test point equal to a data point comes after it
    is_test = order >= n
    steps = [mo._steps(z[order]) for mo in models]
    A = np.stack([s[0] for s in steps], axis=1)             # (M, B, p, p)
    Q = np.stack([s[1] for s in steps], axis=1)
    At = np.swapaxes(A, 2, 3)
    s2 = np.stack([mo.s2 for mo in models], axis=1)         # (n, B)
    S = np.zeros((n, B), dtype=LD)
    G = np.zeros((n, B, p), dtype=LD)
    W = np.zeros((n, B, k), dtype=LD)
    Zt = np.zeros((t.size, B, p, p + k), dtype=LD)
    logdet = np.zeros(B, dtype=LD)
    quad = np.zeros((B, k), dtype=LD)
    # Z = [P | m] (B, p, p + k): the filtered covariance and means
    Z = np.zeros((B, p, p + k), dtype=LD)
    Z[:, :, :p] = np.stack([mo.Pinf for mo in models])
    for j in range(order.size):
        i = order[j]
        if j:
            Z = A[j] @ Z
            Z[:, :, :p] = Z[:, :, :p] @ At[j] + Q[j]
        if is_test[j]:
            Zt[i - n] = Z
            continue
        r = h @ Z                        # [h^T P^- | h^T m^-]
        r[:, p:] -= Yk[i]                # [h^T P^- | -v]
        s = r[:, :p] @ h + s2[i]
        g = (Z[:, :, :p] @ h) / s[:, None]
        Z -= g[:, :, None] * r[:, None, :]  # P^- - g h^T P^-,  m^- + g v
        S[i], G[i] = s, g
        W[i] = -r[:, p:] / s[:, None]
        logdet += np.log(s)
        quad += r[:, p:] ** 2 / s[:, None]
    return dict(logdet=logdet, quad=quad, order=order, is_test=is_test, A=A, S=S.T, G=np.swapaxes(G, 0, 1),
                W=np.swapaxes(W, 0, 1), Zt=Zt)


def log_likelihoods(x, members, y):
    """The longdouble log-likelihood of ``y`` under each ``(sigma, terms)`` of ``members``, in one filter loop."""
    models = [StateSpace(x, sigma, terms) for sigma, terms in members]
    f = _forward(models, np.asarray(y, dtype=np.float64).reshape(-1, 1), np.zeros(0))
    return -(models[0].n * np.log(2 * LD(np.pi)) + f["logdet"] + f["quad"][:, 0]) / 2


def grad_fd(member, theta, x, y, which, h=LD(1) / 512):
    """``d log-likelihood / d theta_which`` at ``theta`` (a vector of log parameters) as a central difference with two
    Richardson steps (error O(h^6)): ``member(theta)`` returns the ``(sigma, terms)`` at ``theta``."""
    theta = np.asarray(theta, dtype=LD)
    steps = [h, h / 2, h / 4]
    thetas = []
    for step in steps:
        for sign in (1, -1):
            th = theta.copy()
            th[which] += sign * step
            thetas.append(th)
    ll = log_likelihoods(x, [member(th) for th in thetas], y)
    D = [(ll[2 * q] - ll[2 * q + 1]) / (2 * step) for q, step in enumerate(steps)]
    R1 = [(4 * D[1] - D[0]) / 3, (4 * D[2] - D[1]) / 3]
    return (16 * R1[1] - R1[0]) / 15
