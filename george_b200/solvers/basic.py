# -*- coding: utf-8 -*-
"""
``BasicSolver`` — dense Cholesky on the H100.

Drop-in for the reference's ``src/george/solvers/basic.py:11-121`` (``kernel.get_value`` + ``scipy.linalg.cholesky``
/ ``cho_solve``): same constructor, methods, properties and return shapes, but the kernel matrix is generated,
factorised and solved against entirely on the device (``csrc/kmat.cu`` + ``csrc/dense.cu``) and never visits the host.
A non positive-definite matrix raises ``numpy.linalg.LinAlgError`` exactly like scipy, which ``GP.recompute`` relies on.
"""

import ctypes as C

import numpy as np

from .. import _lib
from .._spec import DimensionMismatch, flatten, num_params

NONFINITE_RHS = "array must not contain infs or NaNs"


def _check_finite(b):
    """The right-hand side check of scipy's ``cho_solve`` (``check_finite=True``), which the reference's solves go
    through: a NaN or infinite entry raises ``ValueError`` instead of returning a NaN solve."""
    if not np.all(np.isfinite(b)):
        raise ValueError(NONFINITE_RHS)

__all__ = ["BasicSolver"]


class _Handle(object):
    """Owns a pointer that the library function ``create`` makes and ``destroy`` frees (a ``bgp_dense_t*`` or the
    ``bgp_dense_batch_t*`` workspace of the ``batch_*`` statics); never pickled."""

    def __init__(self, create, destroy):
        self.lib = _lib.load()
        self.ptr = C.c_void_p()
        self._destroy = getattr(self.lib, destroy)
        _lib.check(getattr(self.lib, create)(C.byref(self.ptr)))

    def __del__(self):
        if getattr(self, "ptr", None) is not None and self.ptr:
            try:
                self._destroy(self.ptr)
            except Exception:  # interpreter shutdown
                pass
            self.ptr = None


# One batch handle per process, parked here rather than on a GP or solver (which therefore pickle as before): its
# workspace is reused by the next batch of the same size.
_batch_handle = None


def _get_batch_handle():
    global _batch_handle
    if _batch_handle is None:
        _batch_handle = _Handle("bgp_dense_batch_create", "bgp_dense_batch_destroy")
    return _batch_handle


def _points(a):
    """``a`` as contiguous float64, a 1-D array as one column."""
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a[:, None] if a.ndim == 1 else a


def _test_points(kernel, xs):
    """``(spec, xs)`` for the ``_*_call`` statics: ``kernel``'s program and the test points as ``(ns, ndim)``."""
    xs = _points(xs)
    spec = flatten(kernel)
    if xs.ndim != 2 or xs.shape[1] != spec.ndim:
        raise DimensionMismatch("dimension mismatch")  # what kernel.get_value(xs, x) raises
    return spec, xs


def _batch_inputs(spec, params, x, yerr, r, xs=None, which=None):
    """``(x, xs, params, yerr, r, which)`` normalised and checked for the ``batch_*`` statics: ``x`` ``(n, ndim)``,
    ``params`` ``(B, num_params(spec))``, ``yerr`` and ``r`` (``None`` allowed) ``(B, n)``, ``which`` (when given)
    ``(P,)``, then the dimension of the program, ``x`` and ``xs`` (when given, ``(ns, ndim)``)."""
    x = _points(x)
    if xs is not None:
        xs = _points(xs)
    params = np.ascontiguousarray(params, dtype=np.float64)
    yerr = np.ascontiguousarray(yerr, dtype=np.float64)
    if r is not None:
        r = np.ascontiguousarray(r, dtype=np.float64)
    if which is not None:
        which = np.ascontiguousarray(which, dtype=np.uint32)
    if x.ndim != 2 or x.shape[0] == 0:
        raise ValueError("x must have shape (n, ndim) with n > 0")
    n, ndim = x.shape
    npar = num_params(spec)
    if params.ndim != 2 or params.shape[1] != npar:
        raise ValueError("params must have shape (B, {0})".format(npar))
    nb = params.shape[0]
    if yerr.shape != (nb, n) or (r is not None and r.shape != (nb, n)):
        raise ValueError("yerr and r must have shape ({0}, {1})".format(nb, n))
    if which is not None and which.shape != (npar,):
        raise ValueError("which must have shape ({0},)".format(npar))
    if ndim != spec.ndim or (xs is not None and (xs.ndim != 2 or xs.shape[1] != ndim)):
        raise DimensionMismatch("dimension mismatch")
    return x, xs, params, yerr, r, which


def _batch_call(name, spec, params, x, yerr, r, *rest):
    """The library's batched entry point ``name`` on the shared workspace, with the members' common arguments followed
    by ``rest`` (``r`` ``None`` passes NULL); nothing for no members."""
    nb, (n, ndim) = params.shape[0], x.shape
    if nb == 0:
        return
    h = _get_batch_handle()
    _lib.check(getattr(h.lib, name)(h.ptr, C.byref(spec), _lib.ptr(params), nb, params.shape[1], _lib.ptr(x), n, ndim,
                                    _lib.ptr(yerr), None if r is None else _lib.ptr(r), *rest))


def _grad_x_terms_call(call, n, ndim, r, which):
    """``(alpha, g, diagA, dx)`` from a ``bgp_*_grad_x_terms`` entry point ``call(which, r, alpha, g, diag, dx)``
    (the handle bound), after the checks of ``BasicSolver.grad_terms``; ``which`` ``None`` passes NULL."""
    r = np.ascontiguousarray(r, dtype=np.float64)
    if r.shape != (n,):
        raise ValueError("dimension mismatch")
    _check_finite(r)
    alpha = np.empty(n, dtype=np.float64)
    diag = np.empty(n, dtype=np.float64)
    dx = np.empty((n, ndim), dtype=np.float64)
    if which is None:
        _lib.check(call(None, _lib.ptr(r), _lib.ptr(alpha), None, _lib.ptr(diag), _lib.ptr(dx)))
        return alpha, np.zeros(0, dtype=np.float64), diag, dx
    which = np.ascontiguousarray(which, dtype=np.uint32)
    g = np.zeros(max(which.size, 1), dtype=np.float64)
    _lib.check(call(_lib.ptr(which), _lib.ptr(r), _lib.ptr(alpha), _lib.ptr(g), _lib.ptr(diag), _lib.ptr(dx)))
    return alpha, g[:which.size], diag, dx


class BasicSolver(object):

    def __init__(self, kernel):
        self.kernel = kernel
        self._computed = False
        self._log_det = None
        self._handle = None
        self._n = 0

    @property
    def computed(self):
        """Has the covariance matrix been built and factorised (by :func:`compute`)?"""
        return self._computed

    @computed.setter
    def computed(self, v):
        self._computed = v

    @property
    def log_determinant(self):
        """log|K|; ``None`` before :func:`compute`."""
        return self._log_det

    @log_determinant.setter
    def log_determinant(self, v):
        self._log_det = v

    def compute(self, x, yerr):
        """Build K(x, x) + diag(yerr^2) on the device and Cholesky-factorise it (basic.py:51-70)."""
        x = _points(x)
        n, ndim = x.shape
        yerr = np.ascontiguousarray(np.broadcast_to(np.asarray(yerr, dtype=np.float64), (n,)))
        spec = flatten(self.kernel)
        if self._handle is None:
            self._handle = _Handle("bgp_dense_create", "bgp_dense_destroy")
        lib = self._handle.lib
        self._computed = False
        _lib.check(lib.bgp_dense_compute(self._handle.ptr, C.byref(spec), _lib.ptr(x), n, ndim, _lib.ptr(yerr)))
        ld = C.c_double()
        _lib.check(lib.bgp_dense_log_determinant(self._handle.ptr, C.byref(ld)))
        self._n, self._ndim = n, ndim
        self._has_inputs = True
        self.log_determinant = ld.value
        self.computed = True

    def _require(self):
        if self._handle is None or not self._computed:
            raise RuntimeError("you must call 'compute' first")

    def apply_inverse(self, y, in_place=False):
        r"""Solve :math:`K\,x = y` for ``y`` of shape ``(n,)`` or ``(n, nrhs)`` (basic.py:72-87)."""
        self._require()
        y = np.asarray(y)
        if in_place and y.dtype == np.float64 and y.flags.f_contiguous and y.flags.writeable:
            b = y
        else:
            b = np.array(y, dtype=np.float64, order="F")
        if b.shape[0] != self._n:
            raise ValueError("dimension mismatch")
        _check_finite(b)
        nrhs = 1 if b.ndim == 1 else int(np.prod(b.shape[1:]))
        _lib.check(self._handle.lib.bgp_dense_apply_inverse(self._handle.ptr, _lib.ptr(b), nrhs, self._n))
        if in_place and b is not y:
            y[...] = b
            return y
        return b

    def dot_solve(self, y):
        r"""``y^T K^{-1} y`` (basic.py:89-102)."""
        self._require()
        y = np.ascontiguousarray(y, dtype=np.float64)
        if y.shape != (self._n,):
            raise ValueError("dimension mismatch")
        _check_finite(y)
        out = C.c_double()
        _lib.check(self._handle.lib.bgp_dense_dot_solve(self._handle.ptr, _lib.ptr(y), C.byref(out)))
        return out.value

    def apply_sqrt(self, r):
        """``r @ U`` with ``U`` the upper Cholesky factor (basic.py:104-114)."""
        self._require()
        r = np.ascontiguousarray(r, dtype=np.float64)
        r2 = r.reshape(-1, self._n)
        out = np.empty_like(r2)
        _lib.check(self._handle.lib.bgp_dense_apply_sqrt(self._handle.ptr, _lib.ptr(r2), r2.shape[0], _lib.ptr(out)))
        return out.reshape(r.shape)

    def get_inverse(self):
        """Dense ``K^{-1}`` (used by the gradient; basic.py:116-121)."""
        self._require()
        out = np.empty((self._n, self._n), dtype=np.float64)
        _lib.check(self._handle.lib.bgp_dense_get_inverse(self._handle.ptr, _lib.ptr(out)))
        return out

    def grad_terms(self, r, which):
        """``(alpha, g, diagA)`` for ``GP.grad_log_likelihood`` (gp.py:406-468), all computed on the device from the
        stored factor: ``alpha = K^-1 r``, ``g[p] = sum_ij (alpha alpha^T - K^-1)_ij dK_ij/dtheta_p`` over ALL kernel
        parameters (zeros where ``which`` is 0) and ``diagA = diag(alpha alpha^T - K^-1)``.  Replaces
        ``get_inverse()`` + ``kernel.get_gradient`` + ``einsum`` on the host.  Returns ``None`` for a solver restored from
        a pickle (its device handle holds the factor but neither kernel nor coordinates): the caller then composes the
        same quantities from ``get_inverse`` and ``KernelInterface.gradient_contract``."""
        self._require()
        if not getattr(self, "_has_inputs", True):
            return None
        r = np.ascontiguousarray(r, dtype=np.float64)
        if r.shape != (self._n,):
            raise ValueError("dimension mismatch")
        _check_finite(r)
        which = np.ascontiguousarray(which, dtype=np.uint32)
        alpha = np.empty(self._n, dtype=np.float64)
        g = np.zeros(max(which.size, 1), dtype=np.float64)
        diag = np.empty(self._n, dtype=np.float64)
        _lib.check(self._grad_terms_call(_lib.ptr(which), _lib.ptr(r), _lib.ptr(alpha), _lib.ptr(g), _lib.ptr(diag)))
        return alpha, g[:which.size], diag

    def _grad_terms_call(self, which, r, alpha, g, diag):
        return self._handle.lib.bgp_dense_grad_terms(self._handle.ptr, which, r, alpha, g, diag)

    def grad_x_terms(self, r, which):
        """:func:`grad_terms` with the gradient of the log-likelihood with respect to the training inputs, from the
        same pass (``include/bgp.h: bgp_dense_grad_x_terms``): ``(alpha, g, diagA, dx)``, ``alpha``, ``g`` and ``diagA``
        bit for bit what :func:`grad_terms` returns and ``dx[i, q] = sum_j (alpha alpha^T - K^-1)_ij dk(x_i, x_j) /
        dx_iq`` (``(n, ndim)``).  ``which`` ``None`` skips the parameter contraction (``g`` is then empty).  Returns
        ``None`` for a solver restored from a pickle, as :func:`grad_terms` does."""
        self._require()
        if not getattr(self, "_has_inputs", True):
            return None
        return _grad_x_terms_call(self._grad_x_terms_lib, self._n, self._ndim, r, which)

    def _grad_x_terms_lib(self, *args):
        return self._handle.lib.bgp_dense_grad_x_terms(self._handle.ptr, *args)

    def fisher_terms(self, r, which, v, prod_ms=None):
        """The rows of ``GP.fisher_information`` on the device from the stored factor and the resident ``K^-1``
        (``include/bgp.h: bgp_dense_fisher_terms``): ``(grad_terms, rows, rdiag)``.  ``rows`` is ``(nrow, P)`` and
        ``rdiag`` ``(nrow, n)``, one row for each kernel parameter where ``which`` (a 0/1 mask over ALL kernel
        parameters) is set, then one per white-noise vector of ``v`` (``(nv, n)``); with ``B = K^-1 dK K^-1`` for that
        row's ``dK`` (``diag(v_k)`` for a white-noise row), ``rows[., q] = sum_ij B_ij dK_q,ij`` and ``rdiag = diag(B)``.
        ``grad_terms`` is what :func:`grad_terms` returns, bit for bit, when ``r`` is given and ``None`` when ``r`` is
        ``None``.  ``prod_ms`` (an ``(nrow,)`` float64 array) receives each row's product time in ms.  Returns ``None``
        for a solver restored from a pickle, as :func:`grad_terms` does."""
        self._require()
        if not getattr(self, "_has_inputs", True):
            return None
        n = self._n
        which = np.ascontiguousarray(which, dtype=np.uint32)
        v = np.ascontiguousarray(v, dtype=np.float64).reshape(-1, n)
        nrow = int(np.count_nonzero(which)) + v.shape[0]
        rows = np.zeros((nrow, max(which.size, 1)), dtype=np.float64)
        rdiag = np.empty((nrow, n), dtype=np.float64)
        if prod_ms is not None and (prod_ms.shape != (nrow,) or prod_ms.dtype != np.float64):
            raise ValueError("prod_ms must be a float64 array of shape ({0},)".format(nrow))
        terms = None
        rp = alpha = g = diag = None
        if r is not None:
            r = np.ascontiguousarray(r, dtype=np.float64)
            if r.shape != (n,):
                raise ValueError("dimension mismatch")
            _check_finite(r)
            alpha = np.empty(n, dtype=np.float64)
            g = np.zeros(max(which.size, 1), dtype=np.float64)
            diag = np.empty(n, dtype=np.float64)
            rp = _lib.ptr(r)
            terms = alpha, g[:which.size], diag
        _lib.check(self._handle.lib.bgp_dense_fisher_terms(
            self._handle.ptr, _lib.ptr(which), rp, _lib.ptr(v) if v.shape[0] else None, v.shape[0],
            None if alpha is None else _lib.ptr(alpha), None if g is None else _lib.ptr(g),
            None if diag is None else _lib.ptr(diag), _lib.ptr(rows), _lib.ptr(rdiag),
            None if prod_ms is None else _lib.ptr(prod_ms)))
        return terms, rows[:, :which.size], rdiag

    def loo_terms(self, r, which=None):
        """The leave-one-out cross-validation terms of ``GP.loo_*`` on the device from the stored factor
        (``include/bgp.h: bgp_dense_loo_terms``): ``(alpha, d)`` with ``alpha = K^-1 r`` and ``d = diag(K^-1)``; with
        ``which`` (a 0/1 mask over ALL kernel parameters) also ``beta = K^-1 (alpha / d)``, ``g[p] = sum_ij A_ij
        dK_ij/dtheta_p`` (zeros where ``which`` is 0) and ``diagA = diag(A)``, where ``A = 1/2 (beta alpha^T + alpha
        beta^T) - K^-1 diag(c) K^-1`` and ``c = (1 + alpha**2 / d) / (2 d)``.  A gradient with a ``d_i`` that is not
        finite and positive raises ``ValueError`` naming the point.  Returns ``None`` for a solver restored from a pickle,
        as :func:`grad_terms` does."""
        self._require()
        if not getattr(self, "_has_inputs", True):
            return None
        r = np.ascontiguousarray(r, dtype=np.float64)
        if r.shape != (self._n,):
            raise ValueError("dimension mismatch")
        _check_finite(r)
        n = self._n
        alpha = np.empty(n, dtype=np.float64)
        d = np.empty(n, dtype=np.float64)
        if which is None:
            _lib.check(self._loo_terms_call(None, _lib.ptr(r), _lib.ptr(alpha), _lib.ptr(d), None, None, None))
            return alpha, d
        which = np.ascontiguousarray(which, dtype=np.uint32)
        beta = np.empty(n, dtype=np.float64)
        g = np.zeros(max(which.size, 1), dtype=np.float64)
        diag = np.empty(n, dtype=np.float64)
        _lib.check(self._loo_terms_call(_lib.ptr(which), _lib.ptr(r), _lib.ptr(alpha), _lib.ptr(d), _lib.ptr(beta),
                                        _lib.ptr(g), _lib.ptr(diag)))
        return alpha, d, beta, g[:which.size], diag

    def _loo_terms_call(self, which, r, alpha, d, beta, g, diag):
        return self._handle.lib.bgp_dense_loo_terms(self._handle.ptr, which, r, alpha, d, beta, g, diag)

    def predictive(self, kernel, xs, what):
        """The predictive variance (``what="var"``, shape ``(ns,)``) or covariance (``what="cov"``, ``(ns, ns)``) of
        ``GP.predict`` (gp.py:534-545) at ``xs`` (``(ns, ndim)``), computed on the device from the stored factor with
        ``kernel`` for K(x*, x) and K(x*, x*); neither K(x*, x) nor K^-1 K(x, x*) visits the host
        (``include/bgp.h: bgp_dense_predict``).  Returns ``None`` for a solver restored from a pickle (it holds no
        coordinates): the caller then takes the host path."""
        self._require()
        if not getattr(self, "_has_inputs", True):
            return None
        return self._predictive_call(self._handle.lib.bgp_dense_predict, self._handle.ptr, kernel, xs, what)

    @staticmethod
    def _predictive_call(fn, ptr, kernel, xs, what):
        kinds = {"var": _lib.BGP_PREDICT_VAR, "cov": _lib.BGP_PREDICT_COV}
        if what not in kinds:
            raise ValueError("what must be 'var' or 'cov'")
        spec, xs = _test_points(kernel, xs)
        ns = xs.shape[0]
        out = np.empty((ns,) if what == "var" else (ns, ns), dtype=np.float64)
        _lib.check(fn(ptr, C.byref(spec), _lib.ptr(xs), ns, kinds[what], _lib.ptr(out)))
        return out

    def predictive_grad(self, kernel, xs):
        """``(var, dvar)`` for ``GP.grad_predict``: ``var`` (``(ns,)``) is bit for bit :func:`predictive`'s variance
        and ``dvar[j, q] = d var_j / d xs_jq`` (``(ns, ndim)``), both computed on the device from the stored factor
        (``include/bgp.h: bgp_dense_predict_grad``).  Returns ``None`` for a solver restored from a pickle (it holds no
        coordinates): the caller then takes the host path."""
        self._require()
        if not getattr(self, "_has_inputs", True):
            return None
        return self._predictive_grad_call(self._handle.lib.bgp_dense_predict_grad, self._handle.ptr, kernel, xs)

    @staticmethod
    def _predictive_grad_call(fn, ptr, kernel, xs):
        spec, xs = _test_points(kernel, xs)
        ns = xs.shape[0]
        var = np.empty(ns, dtype=np.float64)
        dvar = np.empty((ns, spec.ndim), dtype=np.float64)
        _lib.check(fn(ptr, C.byref(spec), _lib.ptr(xs), ns, _lib.ptr(var), _lib.ptr(dvar)))
        return var, dvar

    def sample_predictive(self, kernel, xs, mean, z, jitter):
        """``mean + z @ L.T`` (``(size, ns)``) with ``L`` the lower Cholesky factor of ``sym(C) + jitter * I``, ``C``
        the covariance :func:`predictive` returns for ``kernel`` at ``xs``: ``GP.sample_conditional``'s draws, with
        ``C`` built, factorised and multiplied on the device without visiting the host
        (``include/bgp.h: bgp_dense_sample``).  ``z``: ``(size, ns)`` standard normals.  Raises
        ``numpy.linalg.LinAlgError`` when that matrix is not positive definite.  Returns ``None`` for a solver restored
        from a pickle (it holds no coordinates): the caller then samples from the host's covariance."""
        self._require()
        if not getattr(self, "_has_inputs", True):
            return None
        return self._sample_call(self._handle.lib.bgp_dense_sample, self._handle.ptr, kernel, xs, mean, z, jitter)

    @staticmethod
    def _sample_call(fn, ptr, kernel, xs, mean, z, jitter):
        spec, xs = _test_points(kernel, xs)
        ns = xs.shape[0]
        mean = np.ascontiguousarray(mean, dtype=np.float64)
        z = np.ascontiguousarray(z, dtype=np.float64)
        if mean.shape != (ns,) or z.ndim != 2 or z.shape[1] != ns:
            raise ValueError("mean must have shape ({0},) and z (size, {0})".format(ns))
        out = np.empty(z.shape, dtype=np.float64)
        _lib.check(fn(ptr, C.byref(spec), _lib.ptr(xs), ns, _lib.ptr(mean), _lib.ptr(z), z.shape[0], float(jitter),
                      _lib.ptr(out)))
        return out

    @staticmethod
    def batch_log_likelihood(spec, params, x, yerr, r):
        """``(log_det, quad, info)``, each ``(B,)``, for ``B`` parameter vectors of one kernel program on the same
        ``x``: member ``b`` factorises ``K(x, x; spec patched with params[b]) + diag(yerr[b]^2)`` and solves against
        ``r[b]`` (``include/bgp.h: bgp_dense_batch_log_likelihood``).  ``info[b]`` is 0, the leading-minor index of a
        matrix that is not positive definite, or -1 when member ``b``'s program fails validation; ``log_det`` and
        ``quad`` are NaN there.  ``spec`` is a :func:`flatten` result, ``params`` ``(B, num_params(spec))``, ``x``
        ``(n,)`` or ``(n, ndim)``, ``yerr`` and ``r`` ``(B, n)``.  The members run in chunks on the device; a
        member's ``log_det`` is bit-identical to :attr:`log_determinant` after :func:`compute` with its spec and
        yerr."""
        x, _, params, yerr, r, _ = _batch_inputs(spec, params, x, yerr, r)
        nb = params.shape[0]
        log_det = np.empty(nb, dtype=np.float64)
        quad = np.empty(nb, dtype=np.float64)
        info = np.zeros(nb, dtype=np.int32)
        _batch_call("bgp_dense_batch_log_likelihood", spec, params, x, yerr, r, _lib.ptr(log_det), _lib.ptr(quad),
                    _lib.ptr(info))
        return log_det, quad, info

    @staticmethod
    def batch_grad_terms(spec, params, x, yerr, r, which):
        """``(log_det, quad, alpha, g, diag, info)`` for ``B`` parameter vectors of one kernel program on the same
        ``x``: member ``b`` factorises as in :func:`batch_log_likelihood` and returns what :func:`grad_terms` returns
        for it, ``alpha`` ``(B, n)``, ``g`` ``(B, P)`` and ``diag`` ``(B, n)``, with ``which`` (``(P,)``) shared by all
        members (``include/bgp.h: bgp_dense_batch_grad_terms``).  ``log_det``, ``quad`` and ``info`` are those of
        :func:`batch_log_likelihood`; a failed member's rows are NaN.  A member's ``alpha``, ``g``, ``diag`` and
        ``log_det`` are bit-identical to :func:`compute` with its spec and yerr followed by :func:`grad_terms`.  More
        than 64 kernel parameters raise ``ValueError`` before anything is solved."""
        x, _, params, yerr, r, which = _batch_inputs(spec, params, x, yerr, r, which=which)
        nb, n, npar = params.shape[0], x.shape[0], params.shape[1]
        log_det = np.empty(nb, dtype=np.float64)
        quad = np.empty(nb, dtype=np.float64)
        alpha = np.empty((nb, n), dtype=np.float64)
        g = np.empty((nb, npar), dtype=np.float64)
        diag = np.empty((nb, n), dtype=np.float64)
        info = np.zeros(nb, dtype=np.int32)
        _batch_call("bgp_dense_batch_grad_terms", spec, params, x, yerr, r, _lib.ptr(which), _lib.ptr(log_det),
                    _lib.ptr(quad), _lib.ptr(alpha), _lib.ptr(diag), _lib.ptr(g), _lib.ptr(info))
        return log_det, quad, alpha, g, diag, info

    @staticmethod
    def batch_loo_terms(spec, params, x, yerr, r, which=None):
        """``(alpha, d, info)``, or with ``which`` (``(P,)``, shared by all members) ``(alpha, d, beta, g, diag,
        info)``, for ``B`` parameter vectors of one kernel program on the same ``x``: member ``b`` factorises as in
        :func:`batch_log_likelihood` and returns what :func:`loo_terms` returns for it, every array but ``g`` (``(B,
        P)``) ``(B, n)`` (``include/bgp.h: bgp_dense_batch_loo_terms``).  ``info`` is that of
        :func:`batch_log_likelihood`; a failed member's rows are NaN.  A member's outputs are bit-identical to
        :func:`compute` with its spec and yerr followed by :func:`loo_terms`, with one difference: a ``d`` that is not
        finite and positive raises nothing here (the member's gradient rows are what that arithmetic gives), so the
        caller checks it.  With ``which``, more than 64 kernel parameters raise ``ValueError`` before anything is
        solved."""
        x, _, params, yerr, r, which = _batch_inputs(spec, params, x, yerr, r, which=which)
        nb, n, npar = params.shape[0], x.shape[0], params.shape[1]
        alpha = np.empty((nb, n), dtype=np.float64)
        d = np.empty((nb, n), dtype=np.float64)
        info = np.zeros(nb, dtype=np.int32)
        if which is None:
            _batch_call("bgp_dense_batch_loo_terms", spec, params, x, yerr, r, None, _lib.ptr(alpha), _lib.ptr(d), None,
                        None, None, _lib.ptr(info))
            return alpha, d, info
        beta = np.empty((nb, n), dtype=np.float64)
        g = np.empty((nb, npar), dtype=np.float64)
        diag = np.empty((nb, n), dtype=np.float64)
        _batch_call("bgp_dense_batch_loo_terms", spec, params, x, yerr, r, _lib.ptr(which), _lib.ptr(alpha),
                    _lib.ptr(d), _lib.ptr(beta), _lib.ptr(g), _lib.ptr(diag), _lib.ptr(info))
        return alpha, d, beta, g, diag, info

    @staticmethod
    def batch_fisher_terms(spec, params, x, yerr, r, which, v, dmu):
        """``(grad_terms, rows, rdiag, kdmu, info)`` for ``B`` parameter vectors of one kernel program on the same
        ``x``: member ``b`` factorises as in :func:`batch_log_likelihood` and returns what :func:`fisher_terms` returns
        for it with ``which`` (``(P,)``, shared by all members) and its white-noise vectors ``v[b]`` (``v`` ``(B, nv,
        n)``), ``rows`` ``(B, nrow, P)`` and ``rdiag`` ``(B, nrow, n)``, plus ``kdmu[b] = K_b^-1 dmu[b]^T`` stored as
        ``(nm, n)`` for its mean gradients ``dmu[b]`` (``dmu`` ``(B, nm, n)``), the solve of ``apply_inverse``
        (``include/bgp.h: bgp_dense_batch_fisher_terms``).  ``grad_terms`` is ``(alpha, g, diag)`` as
        :func:`batch_grad_terms` returns them when ``r`` (``(B, n)``) is given and ``None`` when ``r`` is ``None``.
        ``info`` is that of :func:`batch_log_likelihood`; a failed member's rows are NaN.  A member's outputs are
        bit-identical to :func:`compute` with its spec and yerr followed by :func:`fisher_terms` and
        ``apply_inverse(dmu[b].T)``.  More than 64 kernel parameters raise ``ValueError`` before anything is solved."""
        x, _, params, yerr, r, which = _batch_inputs(spec, params, x, yerr, r, which=which)
        nb, n, npar = params.shape[0], x.shape[0], params.shape[1]
        v = np.ascontiguousarray(v, dtype=np.float64)
        dmu = np.ascontiguousarray(dmu, dtype=np.float64)
        if v.ndim != 3 or v.shape[0] != nb or v.shape[2] != n or dmu.ndim != 3 or dmu.shape[0] != nb or \
                dmu.shape[2] != n:
            raise ValueError("v and dmu must have shape ({0}, nv, {1}) and ({0}, nm, {1})".format(nb, n))
        nv, nm = v.shape[1], dmu.shape[1]
        nrow = int(np.count_nonzero(which)) + nv
        rows = np.empty((nb, nrow, npar), dtype=np.float64)
        rdiag = np.empty((nb, nrow, n), dtype=np.float64)
        kdmu = np.empty((nb, nm, n), dtype=np.float64)
        info = np.zeros(nb, dtype=np.int32)
        terms = (None, None, None)
        if r is not None:
            terms = (np.empty((nb, n), dtype=np.float64), np.empty((nb, npar), dtype=np.float64),
                     np.empty((nb, n), dtype=np.float64))
        _batch_call("bgp_dense_batch_fisher_terms", spec, params, x, yerr, r, _lib.ptr(which),
                    _lib.ptr(v) if nv else None, nv, _lib.ptr(dmu) if nm else None, nm,
                    *[None if t is None else _lib.ptr(t) for t in terms], _lib.ptr(rows), _lib.ptr(rdiag),
                    _lib.ptr(kdmu), _lib.ptr(info))
        return (None if r is None else terms), rows, rdiag, kdmu, info

    @staticmethod
    def batch_predict(spec, params, x, yerr, r, xs, what):
        """``(mean, out, info)`` for ``B`` parameter vectors of one kernel program on the same ``x``: member ``b``
        factorises as in :func:`batch_log_likelihood`, ``mean[b] = K_b(xs, x) K_b^-1 r[b]`` (``(B, ns)``, the kernel
        part of ``GP.predict``'s mean), ``out`` is ``None`` (``what=None``), the variances (``"var"``, ``(B, ns)``) or
        the covariances (``"cov"``, ``(B, ns, ns)``) of :func:`predictive` (``include/bgp.h: bgp_dense_batch_predict``).
        ``info`` is that of :func:`batch_log_likelihood`; a failed member's rows are NaN.  Every entry is bit-identical
        to :func:`compute` with member ``b``'s spec and yerr followed by ``apply_inverse(r[b])``, ``kernel.matvec`` and
        :func:`predictive`.  ``xs``: ``(ns,)`` or ``(ns, ndim)``."""
        kinds = {None: 0, "var": _lib.BGP_PREDICT_VAR, "cov": _lib.BGP_PREDICT_COV}
        if what not in kinds:
            raise ValueError("what must be None, 'var' or 'cov'")
        x, xs, params, yerr, r, _ = _batch_inputs(spec, params, x, yerr, r, xs=xs)
        nb, ns = params.shape[0], xs.shape[0]
        mean = np.empty((nb, ns), dtype=np.float64)
        out = None
        if what == "var":
            out = np.empty((nb, ns), dtype=np.float64)
        elif what == "cov":
            out = np.empty((nb, ns, ns), dtype=np.float64)
        info = np.zeros(nb, dtype=np.int32)
        _batch_call("bgp_dense_batch_predict", spec, params, x, yerr, r, _lib.ptr(xs), ns, kinds[what], _lib.ptr(mean),
                    _lib.ptr(out) if out is not None else None, _lib.ptr(info))
        return mean, out, info

    @staticmethod
    def batch_predict_grad(spec, params, x, yerr, r, xs, return_var):
        """``(mean, var, dmu, dvar, info)`` for ``B`` parameter vectors of one kernel program on the same ``x``: member
        ``b`` factorises as in :func:`batch_log_likelihood`; ``mean`` (``(B, ns)``) is :func:`batch_predict`'s,
        ``dmu[b]`` (``(B, ns, ndim)``) the contraction ``kernel.x1_gradient_matvec(xs, x, K_b^-1 r[b])`` and, with
        ``return_var``, ``var`` (``(B, ns)``) and ``dvar`` (``(B, ns, ndim)``) are what :func:`predictive_grad` returns
        for the member; otherwise both are ``None`` (``include/bgp.h: bgp_dense_batch_predict_grad``).  ``info`` is that
        of :func:`batch_log_likelihood`; a failed member's rows are NaN.  Every entry is bit-identical to
        :func:`compute` with member ``b``'s spec and yerr followed by ``apply_inverse(r[b])``, ``kernel.matvec``,
        ``kernel.x1_gradient_matvec`` and :func:`predictive_grad`.  ``xs``: ``(ns,)`` or ``(ns, ndim)``."""
        x, xs, params, yerr, r, _ = _batch_inputs(spec, params, x, yerr, r, xs=xs)
        nb, (ns, ndim) = params.shape[0], xs.shape
        mean = np.empty((nb, ns), dtype=np.float64)
        dmu = np.empty((nb, ns, ndim), dtype=np.float64)
        var = np.empty((nb, ns), dtype=np.float64) if return_var else None
        dvar = np.empty((nb, ns, ndim), dtype=np.float64) if return_var else None
        info = np.zeros(nb, dtype=np.int32)
        _batch_call("bgp_dense_batch_predict_grad", spec, params, x, yerr, r, _lib.ptr(xs), ns, 1 if return_var else 0,
                    _lib.ptr(mean), _lib.ptr(dmu), _lib.ptr(var) if return_var else None,
                    _lib.ptr(dvar) if return_var else None, _lib.ptr(info))
        return mean, var, dmu, dvar, info

    @staticmethod
    def batch_sample(spec, params, x, yerr, r, xs, mean_add, z, jitter):
        """``(draws, info, draw_info)`` for ``B`` parameter vectors of one kernel program on the same ``x``: member
        ``b`` factorises as in :func:`batch_log_likelihood` and draws ``mu_b + z[b] @ L_b.T`` (``(B, size, ns)``) as
        :func:`sample_predictive` does, ``mu_b`` being the kernel part of ``GP.predict``'s mean plus ``mean_add[b]``
        and ``L_b`` the lower Cholesky factor of ``sym(C_b) + jitter * I`` with ``C_b`` the member's predictive
        covariance (``include/bgp.h: bgp_dense_batch_sample``).  ``info`` is that of :func:`batch_log_likelihood`;
        ``draw_info[b]`` is 0 or the leading minor of that matrix which is not positive definite (0 where ``info[b]``
        is not); a failed member's draws are NaN.  Every draw is bit-identical to :func:`compute` with member ``b``'s
        spec and yerr followed by :func:`sample_predictive`.  ``xs``: ``(ns,)`` or ``(ns, ndim)``; ``mean_add``:
        ``(B, ns)``; ``z``: ``(B, size, ns)`` standard normals."""
        x, xs, params, yerr, r, _ = _batch_inputs(spec, params, x, yerr, r, xs=xs)
        mean_add = np.ascontiguousarray(mean_add, dtype=np.float64)
        z = np.ascontiguousarray(z, dtype=np.float64)
        nb, ns = params.shape[0], xs.shape[0]
        if mean_add.shape != (nb, ns) or z.ndim != 3 or z.shape[0] != nb or z.shape[2] != ns:
            raise ValueError("mean_add must have shape ({0}, {1}) and z ({0}, size, {1})".format(nb, ns))
        draws = np.empty(z.shape, dtype=np.float64)
        info = np.zeros(nb, dtype=np.int32)
        draw_info = np.zeros(nb, dtype=np.int32)
        _batch_call("bgp_dense_batch_sample", spec, params, x, yerr, r, _lib.ptr(xs), ns, _lib.ptr(mean_add), _lib.ptr(z),
                    z.shape[1], float(jitter), _lib.ptr(draws), _lib.ptr(info), _lib.ptr(draw_info))
        return draws, info, draw_info

    # Device handles cannot be pickled.  Like the reference (which pickles its numpy factor, tests/test_pickle.py:21-36:
    # "Unpickled GP shouldn't need to be computed") the Cholesky factor travels with the pickle and is re-uploaded.
    def __getstate__(self):
        state = self.__dict__.copy()
        state["_handle"] = None
        if self._handle is not None and self._computed:
            factor = np.empty((self._n, self._n), dtype=np.float64)
            _lib.check(self._handle.lib.bgp_dense_export_factor(self._handle.ptr, _lib.ptr(factor)))
            state["_pickled_factor"] = factor
        else:
            state["_computed"] = False
        return state

    def __setstate__(self, state):
        factor = state.pop("_pickled_factor", None)
        self.__dict__.update(state)
        self._handle = None
        if factor is not None:
            self._has_inputs = False
            try:
                self._handle = _Handle("bgp_dense_create", "bgp_dense_destroy")
                _lib.check(self._handle.lib.bgp_dense_import_factor(self._handle.ptr, _lib.ptr(factor), self._n,
                                                                   float(self._log_det)))
            except Exception:  # no device where it was unpickled: refactorise lazily on first use
                self._handle = None
                self._computed = False
