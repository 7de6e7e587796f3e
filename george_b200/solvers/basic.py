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


class _DenseHandle(object):
    """Owns a ``bgp_dense_t*``; never pickled."""

    def __init__(self):
        self.lib = _lib.load()
        self.ptr = C.c_void_p()
        _lib.check(self.lib.bgp_dense_create(C.byref(self.ptr)))

    def __del__(self):
        if getattr(self, "ptr", None) is not None and self.ptr:
            self.lib.bgp_dense_destroy(self.ptr)
            self.ptr = None


class _BatchHandle(object):
    """Owns a ``bgp_dense_batch_t*`` (device workspace of ``BasicSolver.batch_log_likelihood`` / ``batch_predict``)."""

    def __init__(self):
        self.lib = _lib.load()
        self.ptr = C.c_void_p()
        _lib.check(self.lib.bgp_dense_batch_create(C.byref(self.ptr)))

    def __del__(self):
        if getattr(self, "ptr", None) is not None and self.ptr:
            try:
                self.lib.bgp_dense_batch_destroy(self.ptr)
            except Exception:  # interpreter shutdown
                pass
            self.ptr = None


# One batch handle per process, parked here rather than on a GP or solver (which therefore pickle as before): its
# workspace is reused by the next batch of the same size.
_batch_handle = None


def _get_batch_handle():
    global _batch_handle
    if _batch_handle is None:
        _batch_handle = _BatchHandle()
    return _batch_handle


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
        x = np.ascontiguousarray(x, dtype=np.float64)
        if x.ndim == 1:
            x = x[:, None]
        n, ndim = x.shape
        yerr = np.ascontiguousarray(np.broadcast_to(np.asarray(yerr, dtype=np.float64), (n,)))
        spec = flatten(self.kernel)
        if self._handle is None:
            self._handle = _DenseHandle()
        lib = self._handle.lib
        self._computed = False
        _lib.check(lib.bgp_dense_compute(self._handle.ptr, C.byref(spec), _lib.ptr(x), n, ndim, _lib.ptr(yerr)))
        ld = C.c_double()
        _lib.check(lib.bgp_dense_log_determinant(self._handle.ptr, C.byref(ld)))
        self._n = n
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
        xs = np.ascontiguousarray(xs, dtype=np.float64)
        if xs.ndim == 1:
            xs = xs[:, None]
        spec = flatten(kernel)
        if xs.ndim != 2 or xs.shape[1] != spec.ndim:
            raise DimensionMismatch("dimension mismatch")  # what kernel.get_value(xs, x) raises
        ns = xs.shape[0]
        out = np.empty((ns,) if what == "var" else (ns, ns), dtype=np.float64)
        _lib.check(fn(ptr, C.byref(spec), _lib.ptr(xs), ns, kinds[what], _lib.ptr(out)))
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
        x = np.ascontiguousarray(x, dtype=np.float64)
        if x.ndim == 1:
            x = x[:, None]
        params = np.ascontiguousarray(params, dtype=np.float64)
        yerr = np.ascontiguousarray(yerr, dtype=np.float64)
        r = np.ascontiguousarray(r, dtype=np.float64)
        if x.ndim != 2 or x.shape[0] == 0:
            raise ValueError("x must have shape (n, ndim) with n > 0")
        n, ndim = x.shape
        if params.ndim != 2 or params.shape[1] != num_params(spec):
            raise ValueError("params must have shape (B, {0})".format(num_params(spec)))
        nb = params.shape[0]
        if yerr.shape != (nb, n) or r.shape != (nb, n):
            raise ValueError("yerr and r must have shape ({0}, {1})".format(nb, n))
        if ndim != spec.ndim:
            raise DimensionMismatch("dimension mismatch")
        log_det = np.empty(nb, dtype=np.float64)
        quad = np.empty(nb, dtype=np.float64)
        info = np.zeros(nb, dtype=np.int32)
        if nb == 0:
            return log_det, quad, info
        h = _get_batch_handle()
        _lib.check(h.lib.bgp_dense_batch_log_likelihood(
            h.ptr, C.byref(spec), _lib.ptr(params), nb, params.shape[1], _lib.ptr(x), n, ndim, _lib.ptr(yerr),
            _lib.ptr(r), _lib.ptr(log_det), _lib.ptr(quad), _lib.ptr(info)))
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
        x = np.ascontiguousarray(x, dtype=np.float64)
        if x.ndim == 1:
            x = x[:, None]
        params = np.ascontiguousarray(params, dtype=np.float64)
        yerr = np.ascontiguousarray(yerr, dtype=np.float64)
        r = np.ascontiguousarray(r, dtype=np.float64)
        which = np.ascontiguousarray(which, dtype=np.uint32)
        if x.ndim != 2 or x.shape[0] == 0:
            raise ValueError("x must have shape (n, ndim) with n > 0")
        n, ndim = x.shape
        npar = num_params(spec)
        if params.ndim != 2 or params.shape[1] != npar:
            raise ValueError("params must have shape (B, {0})".format(npar))
        nb = params.shape[0]
        if yerr.shape != (nb, n) or r.shape != (nb, n):
            raise ValueError("yerr and r must have shape ({0}, {1})".format(nb, n))
        if which.shape != (npar,):
            raise ValueError("which must have shape ({0},)".format(npar))
        if ndim != spec.ndim:
            raise DimensionMismatch("dimension mismatch")
        log_det = np.empty(nb, dtype=np.float64)
        quad = np.empty(nb, dtype=np.float64)
        alpha = np.empty((nb, n), dtype=np.float64)
        g = np.empty((nb, npar), dtype=np.float64)
        diag = np.empty((nb, n), dtype=np.float64)
        info = np.zeros(nb, dtype=np.int32)
        if nb == 0:
            return log_det, quad, alpha, g, diag, info
        h = _get_batch_handle()
        _lib.check(h.lib.bgp_dense_batch_grad_terms(
            h.ptr, C.byref(spec), _lib.ptr(params), nb, npar, _lib.ptr(x), n, ndim, _lib.ptr(yerr), _lib.ptr(r),
            _lib.ptr(which), _lib.ptr(log_det), _lib.ptr(quad), _lib.ptr(alpha), _lib.ptr(diag), _lib.ptr(g),
            _lib.ptr(info)))
        return log_det, quad, alpha, g, diag, info

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
        x = np.ascontiguousarray(x, dtype=np.float64)
        if x.ndim == 1:
            x = x[:, None]
        xs = np.ascontiguousarray(xs, dtype=np.float64)
        if xs.ndim == 1:
            xs = xs[:, None]
        params = np.ascontiguousarray(params, dtype=np.float64)
        yerr = np.ascontiguousarray(yerr, dtype=np.float64)
        r = np.ascontiguousarray(r, dtype=np.float64)
        if x.ndim != 2 or x.shape[0] == 0:
            raise ValueError("x must have shape (n, ndim) with n > 0")
        n, ndim = x.shape
        if params.ndim != 2 or params.shape[1] != num_params(spec):
            raise ValueError("params must have shape (B, {0})".format(num_params(spec)))
        nb = params.shape[0]
        if yerr.shape != (nb, n) or r.shape != (nb, n):
            raise ValueError("yerr and r must have shape ({0}, {1})".format(nb, n))
        if ndim != spec.ndim or xs.ndim != 2 or xs.shape[1] != ndim:
            raise DimensionMismatch("dimension mismatch")
        ns = xs.shape[0]
        mean = np.empty((nb, ns), dtype=np.float64)
        out = None
        if what == "var":
            out = np.empty((nb, ns), dtype=np.float64)
        elif what == "cov":
            out = np.empty((nb, ns, ns), dtype=np.float64)
        info = np.zeros(nb, dtype=np.int32)
        if nb == 0:
            return mean, out, info
        h = _get_batch_handle()
        _lib.check(h.lib.bgp_dense_batch_predict(
            h.ptr, C.byref(spec), _lib.ptr(params), nb, params.shape[1], _lib.ptr(x), n, ndim, _lib.ptr(yerr),
            _lib.ptr(r), _lib.ptr(xs), ns, kinds[what], _lib.ptr(mean), _lib.ptr(out) if out is not None else None,
            _lib.ptr(info)))
        return mean, out, info

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
                self._handle = _DenseHandle()
                _lib.check(self._handle.lib.bgp_dense_import_factor(self._handle.ptr, _lib.ptr(factor), self._n,
                                                                   float(self._log_det)))
            except Exception:  # no device where it was unpickled: refactorise lazily on first use
                self._handle = None
                self._computed = False
