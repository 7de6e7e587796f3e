# -*- coding: utf-8 -*-
"""Closed-form references for ``c * ExpKernel(m)`` on sorted 1-D inputs (test infrastructure; numpy only).

On sorted points this covariance is that of an Ornstein-Uhlenbeck process, and its Cholesky factor is known entry by
entry.  Let ``l = sqrt(m)`` (``ExpKernel`` evaluates ``exp(-sqrt(r^2))`` with ``r^2 = (x_i - x_j)^2 / m``),

    K_ij = c exp(-|x_i - x_j| / l),   rho_j = exp(-(x_j - x_{j-1}) / l),   s_0 = 1,   s_j = sqrt(1 - rho_j^2).

Then ``K = L L^T`` with

    L_ij = sqrt(c) exp(-(x_i - x_j) / l) s_j    (i >= j),   0 above the diagonal.

Proof: for i >= k, ``(L L^T)_ik = c exp(-(x_i - x_k) / l) sum_{j <= k} E_j s_j^2`` with
``E_j = exp(-2 (x_k - x_j) / l)``.  Since ``E_j rho_j^2 = E_{j-1}``, each term ``E_j s_j^2 = E_j - E_{j-1}`` for
j >= 1 and ``E_0 s_0^2 = E_0``, so the sum telescopes to ``E_k = 1`` and ``(L L^T)_ik = K_ik``.

Everything else follows in O(n):

* ``log det K = n log c + 2 sum_j log s_j``;
* ``L = sqrt(c) A diag(s)`` with ``A_ij = exp(-(x_i - x_j) / l)`` (i >= j), and ``A^-1`` is unit lower bidiagonal with
  ``-rho_j`` below the diagonal, so ``(L^-1 z)_j = (z_j - rho_j z_{j-1}) / (sqrt(c) s_j)`` and
  ``(L^-T w)_j = (w_j / s_j - rho_{j+1} w_{j+1} / s_{j+1}) / sqrt(c)``;
* ``K^-1 = L^-T L^-1`` is tridiagonal: ``c K^-1_jj = 1 / s_j^2 + rho_{j+1}^2 / s_{j+1}^2`` and
  ``c K^-1_{j,j+1} = -rho_{j+1} / s_{j+1}^2``;
* ``o = z L^T`` is the AR(1) recursion ``o_j = rho_j o_{j-1} + sqrt(c) s_j z_j``;
* for theta = (log c, log m), ``dK/dlog c = K`` and ``dK/dlog m = D / 2`` with ``D_ij = K_ij |x_i - x_j| / l``
  (``d sqrt(r^2) / dlog m = -sqrt(r^2) / 2``).  The gradient terms of ``grad_terms``,
  ``g_p = sum_ij (alpha alpha^T - K^-1)_ij dK_ij/dtheta_p`` with ``alpha = K^-1 r``, are therefore
  ``g_c = r . alpha - n`` and ``g_m = alpha^T D alpha / 2 - tr(K^-1 D) / 2``.  D is semi-separable: ``D a`` takes one
  forward and one backward sweep, and ``tr(K^-1 D)`` needs only the first off-diagonal of K^-1 (D's diagonal is 0);
* the leave-one-out terms of ``loo_terms`` (``loo_terms`` has the derivation): ``K^-1 diag(w) K^-1`` is pentadiagonal,
  and each contraction with K or D is a dot with one ``K a`` / ``D a`` sweep plus five bands;
* the likelihood factors over the points, ``p(r) = prod_j N(r_j; rho_j r_{j-1}, c s_j^2)`` (``factor_terms``), and the
  expected Fisher information (``fisher``) and the gradient in the inputs (``grad_x``) are sums over those factors.

Every recursion runs on the ratios ``rho_j`` and the scaled gaps ``(x_j - x_{j-1}) / l``, never on ``exp(+-x / l)``,
so nothing overflows however long the interval.  All arithmetic is ``np.longdouble`` (x87 80-bit on x86-64, eps
1.1e-19), so for well-conditioned K (gaps of at least 0.2 l give rho <= 0.82 and cond(K) <= 10) the distance of a
float64 result from these values is the float64 result's own error.
"""
import numpy as np

LD = np.longdouble
assert np.finfo(LD).nmant >= 63, (
    "np.longdouble has a {0}-bit mantissa here: the extended-precision reference needs the 80-bit x87 format"
    .format(np.finfo(LD).nmant))

# Test points see the data within this many length scales: a dropped term of the predictive mean or variance is below
# exp(-100) = 3.7e-44 of c, far below longdouble rounding.
PREDICT_WINDOW = 100


class OU(object):
    """The closed forms for ``K = c * ExpKernel(m)`` evaluated at the sorted points ``x`` (``(n,)`` or ``(n, 1)``)."""

    def __init__(self, x, c, m):
        x = np.asarray(x, dtype=np.float64).reshape(-1)
        if x.size > 1 and not np.all(np.diff(x) > 0):
            raise ValueError("x must be strictly increasing")
        self.n = x.size
        self.x = x.astype(LD)
        self.c = LD(c)
        self.ell = np.sqrt(LD(m))
        self.sqrtc = np.sqrt(self.c)
        # delta_j = (x_j - x_{j-1}) / l and rho_j = exp(-delta_j) for j >= 1; delta_0 = rho_0 = 0, s_0 = 1
        self.delta = np.zeros(self.n, dtype=LD)
        self.delta[1:] = np.diff(self.x) / self.ell
        self.rho = np.exp(-self.delta)
        self.rho[0] = 0
        s2 = -np.expm1(-2 * self.delta)  # 1 - rho^2 without cancellation
        s2[0] = 1
        self.s2 = s2
        self.s = np.sqrt(s2)

    # ---- the factor ---------------------------------------------------------------------------------------------
    def logdet(self):
        """``log det K``."""
        return self.n * np.log(self.c) + 2 * np.sum(np.log(self.s))

    def chol_columns(self, cols):
        """``L[:, cols]`` (``(n, len(cols))``), entry by entry."""
        cols = np.asarray(cols, dtype=np.int64)
        out = np.zeros((self.n, cols.size), dtype=LD)
        for k, j in enumerate(cols):
            out[j:, k] = self.sqrtc * self.s[j] * np.exp(-(self.x[j:] - self.x[j]) / self.ell)
        return out

    def inv_chol(self, z):
        """``L^-1 z`` for ``z`` of shape ``(n,)`` or ``(n, k)``."""
        z = np.asarray(z, dtype=LD)
        rho, s = (self.rho, self.s) if z.ndim == 1 else (self.rho[:, None], self.s[:, None])
        prev = np.zeros_like(z)
        prev[1:] = z[:-1]
        return (z - rho * prev) / (self.sqrtc * s)

    def inv_chol_t(self, w):
        """``L^-T w`` for ``w`` of shape ``(n,)`` or ``(n, k)``."""
        w = np.asarray(w, dtype=LD)
        rho, s = (self.rho, self.s) if w.ndim == 1 else (self.rho[:, None], self.s[:, None])
        q = w / s
        nxt = np.zeros_like(q)
        nxt[:-1] = rho[1:] * q[1:]
        return (q - nxt) / self.sqrtc

    def solve(self, b):
        """``K^-1 b`` for ``b`` of shape ``(n,)`` or ``(n, k)``."""
        return self.inv_chol_t(self.inv_chol(b))

    def inv_tridiag(self):
        """``(d, e)``: the diagonal (``(n,)``) and the first off-diagonal (``(n - 1,)``, ``e_j = K^-1_{j,j+1}``) of the
        tridiagonal K^-1."""
        d = 1 / self.s2
        d[:-1] += self.rho[1:] ** 2 / self.s2[1:]
        e = -self.rho[1:] / self.s2[1:]
        return d / self.c, e / self.c

    def sqrt_rows(self, z):
        """``z @ L^T`` for ``z`` of shape ``(n,)`` or ``(k, n)``: the AR(1) recursion, one sweep over the points."""
        z = np.asarray(z, dtype=LD)
        zz = z.reshape(-1, self.n)
        out = np.empty_like(zz)
        o = np.zeros(zz.shape[0], dtype=LD)
        w = self.sqrtc * self.s
        for j in range(self.n):
            o = self.rho[j] * o + w[j] * zz[:, j]
            out[:, j] = o
        return out.reshape(z.shape)

    # ---- the log-likelihood gradient ------------------------------------------------------------------------------
    def _sweeps(self, a):
        """``(K a, D a)`` for a vector ``a``, ``D_ij = K_ij |x_i - x_j| / l``, in one forward and one backward sweep.

        Forward: ``P_i = sum_{j<i} exp(-(x_i - x_j)/l) a_j`` and ``Q_i = sum_{j<i} exp(-(x_i - x_j)/l) (x_i - x_j)/l a_j``
        obey ``P_i = rho_i (P_{i-1} + a_{i-1})`` and ``Q_i = rho_i (Q_{i-1} + delta_i (P_{i-1} + a_{i-1}))``; the
        backward sweep is the mirror image.  ``(K a)_i = c (a_i + P_i + P'_i)`` and ``(D a)_i = c (Q_i + Q'_i)``."""
        a = np.asarray(a, dtype=LD).tolist()
        rho, dl = self.rho.tolist(), self.delta.tolist()
        n = self.n
        ka, da = list(a), [LD(0)] * n
        P = Q = LD(0)
        for i in range(1, n):
            t = P + a[i - 1]
            Q = rho[i] * (Q + dl[i] * t)
            P = rho[i] * t
            ka[i] += P
            da[i] = Q
        P = Q = LD(0)
        for i in range(n - 2, -1, -1):
            t = P + a[i + 1]
            Q = rho[i + 1] * (Q + dl[i + 1] * t)
            P = rho[i + 1] * t
            ka[i] += P
            da[i] += Q
        return self.c * np.array(ka, dtype=LD), self.c * np.array(da, dtype=LD)

    def apply_d(self, a):
        """``D a`` for a vector ``a`` (see ``_sweeps``)."""
        return self._sweeps(a)[1]

    def apply_k(self, a):
        """``K a`` for a vector ``a`` (see ``_sweeps``)."""
        return self._sweeps(a)[0]

    def trace_kinv_d(self):
        """``tr(K^-1 D) = 2 sum_j K^-1_{j,j+1} D_{j,j+1}``, with ``D_{j,j+1} = c rho_{j+1} delta_{j+1}``."""
        _, e = self.inv_tridiag()
        return 2 * np.sum(e * self.c * self.rho[1:] * self.delta[1:])

    def grad_terms(self, r):
        """``(alpha, g, diag)`` of ``grad_terms`` for theta = (log c, log m): ``alpha = K^-1 r``, ``g`` (``(2,)``) and
        ``diag = alpha^2 - diag(K^-1)``."""
        r = np.asarray(r, dtype=LD)
        alpha = self.solve(r)
        g_c = r @ alpha - self.n
        g_m = (alpha @ self.apply_d(alpha) - self.trace_kinv_d()) / 2
        d, _ = self.inv_tridiag()
        return alpha, np.array([g_c, g_m], dtype=LD), alpha ** 2 - d

    # ---- leave-one-out cross-validation -------------------------------------------------------------------------------
    def loo_terms(self, r):
        """The leave-one-out terms of ``loo_terms`` for theta = (log c, log m), as a dict:

        * ``alpha = K^-1 r``, ``d = diag(K^-1) = t`` (the diagonal of the tridiagonal ``T = K^-1``, off-diagonal ``e``);
        * ``beta = K^-1 q`` with ``q = alpha / d``, and the weights ``w_i = (1 + alpha_i q_i) / (2 d_i)``;
        * ``M = T diag(w) T`` is pentadiagonal: ``M_jj = w_{j-1} e_{j-1}^2 + w_j t_j^2 + w_{j+1} e_j^2``,
          ``M_{j,j+1} = e_j (w_j t_j + w_{j+1} t_{j+1})`` and ``M_{j,j+2} = e_j w_{j+1} e_{j+1}``;
        * ``A = 1/2 (beta alpha^T + alpha beta^T) - M``, so ``diagA = alpha beta - diag(M)``;
        * ``g_logc = sum_ij K_ij A_ij = beta . r - sum_j w_j t_j``: ``K alpha = r``, and
          ``tr(K T W T) = tr(W T K T) = tr(W T)``;
        * ``g_logm = sum_ij (D / 2)_ij A_ij = (beta^T D alpha - sum_ij D_ij M_ij) / 2``.  D's diagonal is 0, so the
          second term needs only the bands ``D_{j,j+1} = c rho_{j+1} delta_{j+1}`` and
          ``D_{j,j+2} = c rho_{j+1} rho_{j+2} (delta_{j+1} + delta_{j+2})`` (c the kernel amplitude);
        * ``value = sum_i [-1/2 log 2 pi + 1/2 log d_i - alpha_i^2 / (2 d_i)]``; the LOO predictive of ``r_i`` is
          ``r_i - alpha_i / d_i`` with variance ``1 / d_i``.

        ``gscale`` bounds ``sum_ij |dK_p|_ij |A_ij|`` from above in O(n): K and D have non-negative entries and
        ``|M| <= |T| W |T|`` (five bands, W > 0), so it is ``|beta|^T K |alpha| + sum_ij K_ij (|T| W |T|)_ij`` for log c
        and half of the same with D for log m."""
        r = np.asarray(r, dtype=LD)
        t, e = self.inv_tridiag()
        alpha = self.solve(r)
        d = t.copy()
        q = alpha / d
        beta = self.solve(q)
        w = (1 + alpha * q) / (2 * d)
        # the bands of M = T W T (M1, M2: first and second super-diagonals) and of |T| W |T|
        M0 = w * t * t
        M0[1:] += w[:-1] * e * e
        M0[:-1] += w[1:] * e * e
        M1 = e * (w[:-1] * t[:-1] + w[1:] * t[1:])
        M2 = e[:-1] * w[1:-1] * e[1:]
        # the bands of K / c and of D / c (D0 = 0)
        K1 = self.rho[1:]
        K2 = self.rho[1:-1] * self.rho[2:]
        D1 = self.rho[1:] * self.delta[1:]
        D2 = K2 * (self.delta[1:-1] + self.delta[2:])
        Db = self._sweeps(beta)[1]
        g_c = beta @ r - np.sum(w * t)
        g_m = (Db @ alpha - 2 * self.c * (np.sum(D1 * M1) + np.sum(D2 * M2))) / 2
        value = np.sum(-np.log(2 * LD(np.pi)) / 2 + np.log(d) / 2 - alpha ** 2 / (2 * d))
        aa, ab = np.abs(alpha), np.abs(beta)
        Kab, Dab = self._sweeps(ab)
        band_k = self.c * (np.sum(M0) + 2 * np.sum(K1 * np.abs(M1)) + 2 * np.sum(K2 * np.abs(M2)))
        band_d = 2 * self.c * (np.sum(D1 * np.abs(M1)) + np.sum(D2 * np.abs(M2)))
        gscale = np.array([Kab @ aa + band_k, (Dab @ aa + band_d) / 2], dtype=LD)
        return dict(alpha=alpha, d=d, beta=beta, g=np.array([g_c, g_m], dtype=LD), diagA=alpha * beta - M0,
                    value=value, gscale=gscale)

    # ---- the factors of the likelihood: Fisher information and input gradient -------------------------------------
    def factor_terms(self, r, delta=None):
        """``t_j = log N(r_j; rho_j r_{j-1}, v_j)`` with ``v_0 = c`` and ``v_j = c s_j^2``, so that ``sum_j t_j`` is the
        log-likelihood of ``r`` (``(n,)``).  ``K = L L^T`` with ``L = sqrt(c) A diag(s)`` makes ``L^-1 r`` the scaled
        innovations ``u_j / (sqrt(c) s_j)``, ``u_j = r_j - rho_j r_{j-1}``, and ``log det K`` the sum of ``log v_j``.
        ``delta`` (``(n,)``, entry 0 unused) replaces the scaled gaps: t_j depends on the inputs through delta_j alone."""
        r = np.asarray(r, dtype=LD)
        dl = self.delta if delta is None else np.asarray(delta, dtype=LD)
        rho = np.exp(-dl)
        rho[0] = 0
        v = -self.c * np.expm1(-2 * dl)
        v[0] = self.c
        u = r.copy()
        u[1:] -= rho[1:] * r[:-1]
        return -np.log(2 * LD(np.pi) * v) / 2 - u * u / (2 * v)

    def fisher(self, mean=True):
        """The expected Fisher information for theta = (log c, log m), led by a constant mean's row with ``mean``:
        ``(3, 3)`` in the order (mean, log c, log m), or ``(2, 2)``.

        The factors of ``factor_terms`` have scores of zero conditional mean given the earlier points, so scores of
        different factors are uncorrelated and F sums over the factors.  For ``N(r; rho r', v)`` with ``E[r'^2] = c``
        a factor adds ``c drho_p drho_q / v + dv_p dv_q / (2 v^2)``.  With ``drho_j/dlog m = rho_j delta_j / 2``
        (``delta_j = gap / sqrt(m)``), ``dv_j/dlog m = -c rho_j^2 delta_j``, ``dv_j/dlog c = v_j``, ``drho/dlog c = 0``
        and nothing for factor 0 but its ``log c`` term:

            F_cc = n / 2,   F_cm = -sum_j rho_j^2 delta_j / (2 s_j^2) = tr(K^-1 D) / 4,
            F_mm = sum_j [rho_j^2 delta_j^2 / (4 s_j^2) + rho_j^4 delta_j^2 / (2 s_j^4)].

        The mean enters the mean of r only: ``F_mumu = 1^T K^-1 1``, the sum of the tridiagonal K^-1's entries, and
        its cross terms with the kernel parameters are 0."""
        rho2, dl, s2 = self.rho[1:] ** 2, self.delta[1:], self.s2[1:]
        F = np.zeros((2, 2), dtype=LD)
        F[0, 0] = LD(self.n) / 2
        F[0, 1] = F[1, 0] = -np.sum(rho2 * dl / (2 * s2))
        F[1, 1] = np.sum(rho2 * dl * dl / (4 * s2) + rho2 * rho2 * dl * dl / (2 * s2 * s2))
        if not mean:
            return F
        d, e = self.inv_tridiag()
        out = np.zeros((3, 3), dtype=LD)
        out[0, 0] = np.sum(d) + 2 * np.sum(e)
        out[1:, 1:] = F
        return out

    def grad_x(self, r):
        """``(dx, scale)``: ``dx_i = d log p(r) / d x_i`` (``(n,)``), which is ``sum_j (alpha alpha^T - K^-1)_ij
        dk(x_i, x_j)/dx_i``, and a per-entry bound of what that contraction sums.

        Factor j of ``factor_terms`` depends on the inputs through the gap ``x_j - x_{j-1}`` alone.  With
        ``rho' = -rho_j / l`` and ``v' = 2 c rho_j^2 / l`` its derivatives in the gap, the factor's derivative is

            G_j = -v' / (2 v_j) + u_j r_{j-1} rho' / v_j + u_j^2 v' / (2 v_j^2),

        and x_i is the upper end of gap i and the lower end of gap i + 1: ``dx_i = G_i - G_{i+1}`` (G_0 = G_n = 0),
        which telescopes to ``sum_i dx_i = 0``.

        ``scale_i >= sum_j |A_ij| |dk_ij/dx_i|`` (A = alpha alpha^T - K^-1): ``|dk_ij/dx_i| = k_ij / l`` off the
        diagonal and 0 on it, and K^-1 is tridiagonal, so it is ``|alpha_i| ((K |alpha|)_i - c |alpha_i|) / l`` plus
        ``|K^-1_{i,i+-1}| k_{i,i+-1} / l`` for the two neighbours."""
        r = np.asarray(r, dtype=LD)
        rho, s2, ell, n = self.rho[1:], self.s2[1:], self.ell, self.n
        v = self.c * s2
        u = r[1:] - rho * r[:-1]
        drho = -rho / ell
        dv = 2 * self.c * rho * rho / ell
        G = -dv / (2 * v) + u * r[:-1] * drho / v + u * u * dv / (2 * v * v)
        dx = np.zeros(n, dtype=LD)
        dx[1:] += G
        dx[:-1] -= G
        alpha = self.solve(r)
        aa = np.abs(alpha)
        ka = self.apply_k(aa)
        _, e = self.inv_tridiag()
        nb = np.abs(e) * self.c * rho / ell  # |K^-1_{j,j+1}| |dk_{j,j+1}|
        scale = aa * (ka - self.c * aa) / ell
        scale[1:] += nb
        scale[:-1] += nb
        return dx, scale

    # ---- prediction -------------------------------------------------------------------------------------------------
    def predict(self, t, alpha):
        """``(mean, var)`` at the test points ``t``: ``mean = K(t, x) alpha`` and ``var = c - |w|^2`` with
        ``w = L^-1 K(x, t)``, over the points within ``PREDICT_WINDOW`` length scales of each test point (``w`` is
        exactly 0 past the first point at or above t, and below ``exp(-PREDICT_WINDOW)`` further down)."""
        t = np.asarray(t, dtype=np.float64).reshape(-1)
        alpha = np.asarray(alpha, dtype=LD)
        x64 = self.x.astype(np.float64)
        span = float(PREDICT_WINDOW * self.ell)
        mean = np.empty(t.size, dtype=LD)
        var = np.empty(t.size, dtype=LD)
        for k, tk in enumerate(t):
            lo = int(np.searchsorted(x64, tk - span, side="left"))
            hi = int(np.searchsorted(x64, tk + span, side="right"))
            lo1 = max(lo - 1, 0)
            kt = self.c * np.exp(-np.abs(self.x[lo1:hi] - LD(tk)) / self.ell)  # K(x_j, t) for j in [lo1, hi)
            cur = kt[lo - lo1:]
            prev = np.empty_like(cur)  # K(x_{j-1}, t); rho_0 = 0 makes the first row's value irrelevant
            prev[1:] = cur[:-1]
            prev[0] = kt[0] if lo1 < lo else 0
            w = (cur - self.rho[lo:hi] * prev) / (self.sqrtc * self.s[lo:hi])
            mean[k] = cur @ alpha[lo:hi]
            var[k] = self.c - w @ w
        return mean, var


def exp_problem(n, ell, seed, x0=0.0, gap=(0.2, 1.0)):
    """Sorted points with gaps drawn from ``uniform(*gap) * ell``, starting at ``x0``."""
    rng = np.random.default_rng(seed)
    x = np.empty(n)
    x[0] = x0
    x[1:] = x0 + np.cumsum(rng.uniform(gap[0], gap[1], n - 1) * ell)
    return x
