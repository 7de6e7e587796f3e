# -*- coding: utf-8 -*-
"""
``KernelInterface`` — the evaluation handle behind ``Kernel.get_value`` / ``get_gradient``.

Mirrors the pybind11 class of the reference (``src/george/kernel_interface.cpp:44-167``): constructed from a
kernel-spec object (parameters are snapshotted at construction, as ``parse_kernel_spec`` does), it exposes
``value_general`` / ``value_symmetric`` / ``value_diagonal`` / ``gradient_general`` / ``gradient_symmetric`` with the
reference's shapes, and pickles as its spec.  The arithmetic runs in the fused CUDA kernel-matrix build
(``csrc/kmat.cu``) through the C ABI; there is no CPU path.
"""

import ctypes as C

import numpy as np

from . import _lib
from ._spec import DimensionMismatch, flatten, num_params


def _as2d(x, ndim):
    x = np.ascontiguousarray(x, dtype=np.float64)
    if x.ndim != 2:
        raise ValueError("array has incorrect number of dimensions: {0}; expected 2".format(x.ndim))
    if x.shape[1] != ndim:
        raise DimensionMismatch("dimension mismatch")
    return x


class KernelInterface(object):

    def __init__(self, kernel_spec):
        self._kernel_spec = kernel_spec
        self._spec = flatten(kernel_spec)
        self._size = num_params(self._spec)

    # pickle as the spec object (kernel_interface.cpp:159-167)
    def __getstate__(self):
        return self._kernel_spec

    def __setstate__(self, spec):
        self.__init__(spec)

    @property
    def ndim(self):
        return int(self._spec.ndim)

    @property
    def size(self):
        return self._size

    @property
    def spec(self):
        """The flattened POD program (``include/bgp.h: bgp_kernel_spec_t``)."""
        return self._spec

    def value_general(self, x1, x2):
        x1, x2 = _as2d(x1, self.ndim), _as2d(x2, self.ndim)
        out = np.empty((x1.shape[0], x2.shape[0]), dtype=np.float64)
        lib = _lib.load()
        _lib.check(lib.bgp_kmat_general(C.byref(self._spec), _lib.ptr(x1), x1.shape[0], _lib.ptr(x2), x2.shape[0],
                                        _lib.ptr(out)))
        return out

    def value_symmetric(self, x):
        x = _as2d(x, self.ndim)
        out = np.empty((x.shape[0], x.shape[0]), dtype=np.float64)
        lib = _lib.load()
        _lib.check(lib.bgp_kmat_symmetric(C.byref(self._spec), _lib.ptr(x), x.shape[0], _lib.ptr(out)))
        return out

    def value_diagonal(self, x1, x2):
        x1, x2 = _as2d(x1, self.ndim), _as2d(x2, self.ndim)
        if x1.shape[0] != x2.shape[0]:
            raise DimensionMismatch("dimension mismatch")
        out = np.empty(x1.shape[0], dtype=np.float64)
        lib = _lib.load()
        _lib.check(lib.bgp_kmat_diagonal(C.byref(self._spec), _lib.ptr(x1), _lib.ptr(x2), x1.shape[0], _lib.ptr(out)))
        return out

    def _which(self, which):
        which = np.ascontiguousarray(which, dtype=np.uint32)
        if which.shape != (self._size,):
            raise DimensionMismatch("dimension mismatch")
        return which

    def gradient_general(self, which, x1, x2):
        which = self._which(which)
        x1, x2 = _as2d(x1, self.ndim), _as2d(x2, self.ndim)
        out = np.empty((x1.shape[0], x2.shape[0], self._size), dtype=np.float64)
        lib = _lib.load()
        _lib.check(lib.bgp_kmat_gradient_general(C.byref(self._spec), _lib.ptr(which), _lib.ptr(x1), x1.shape[0],
                                                 _lib.ptr(x2), x2.shape[0], _lib.ptr(out)))
        return out

    def gradient_symmetric(self, which, x):
        which = self._which(which)
        x = _as2d(x, self.ndim)
        out = np.empty((x.shape[0], x.shape[0], self._size), dtype=np.float64)
        lib = _lib.load()
        _lib.check(lib.bgp_kmat_gradient_symmetric(C.byref(self._spec), _lib.ptr(which), _lib.ptr(x), x.shape[0],
                                                   _lib.ptr(out)))
        return out

    # ---- matrix-free consumers (not in the reference: it forms the matrix and calls numpy) --------------------------
    def matvec(self, x1, x2, v, diag=None):
        """``K(x1, x2) @ v`` (plus ``diag * v`` for a square operator) without forming the ``(n1, n2)`` matrix:
        what ``GP.predict`` needs for its mean (reference gp.py:524-528).  ``v``: ``(n2,)`` or ``(n2, k)``."""
        x1, x2 = _as2d(x1, self.ndim), _as2d(x2, self.ndim)
        v = np.asarray(v, dtype=np.float64)
        if v.shape[0] != x2.shape[0] or v.ndim not in (1, 2):
            raise DimensionMismatch("dimension mismatch")
        vf = np.asfortranarray(v.reshape(x2.shape[0], -1))
        out = np.empty((x1.shape[0], vf.shape[1]), dtype=np.float64, order="F")
        d = None
        if diag is not None:
            d = np.ascontiguousarray(diag, dtype=np.float64)
            if d.shape != (x1.shape[0],) or x1.shape[0] != x2.shape[0]:
                raise DimensionMismatch("dimension mismatch")
        same = x1.shape == x2.shape and x1.ctypes.data == x2.ctypes.data  # both C-contiguous here
        _lib.check(_lib.load().bgp_kmat_matvec(C.byref(self._spec), _lib.ptr(x1), x1.shape[0],
                                               _lib.ptr(x1 if same else x2), x2.shape[0],
                                               _lib.ptr(d) if d is not None else None, _lib.ptr(vf), vf.shape[1],
                                               _lib.ptr(out)))
        return out[:, 0].copy() if v.ndim == 1 else out

    def gradient_contract(self, which, x, A):
        """``einsum("ijk,ij", gradient_symmetric(which, x), A)`` without the ``(n, n, P)`` tensor (gp.py:465-466)."""
        which = self._which(which)
        x = _as2d(x, self.ndim)
        A = np.ascontiguousarray(A, dtype=np.float64)
        if A.shape != (x.shape[0], x.shape[0]):
            raise DimensionMismatch("dimension mismatch")
        out = np.zeros(self._size, dtype=np.float64)
        _lib.check(_lib.load().bgp_kmat_gradient_contract(C.byref(self._spec), _lib.ptr(which), _lib.ptr(x), x.shape[0],
                                                          _lib.ptr(A), _lib.ptr(out)))
        return out

    def x1_gradient_matvec(self, x1, x2, v, scale=1.0, add_prior=False):
        """``out[i, q] = (add_prior ? d k(x1_i, x1_i) / d x1_iq : 0) + scale * sum_j d k(x1_i, x2_j) / d x1_iq V_ji``
        (``(n1, ndim)``) without the ``(n1, n2, ndim)`` gradient tensor, ``V_ji = v[j]`` for ``v`` of shape ``(n2,)`` and
        ``v[j, i]`` for ``(n2, n1)``: ``GP.grad_predict``'s ``dmu`` (``v = alpha``) and, with ``scale=-2`` and
        ``add_prior``, its ``dvar`` (``v = K^-1 K(x, x1)``).  True derivatives for every metric, where
        :func:`x1_gradient_general` returns the reference's values (include/bgp.h: bgp_kmat_x1_gradient_matvec)."""
        x1, x2 = _as2d(x1, self.ndim), _as2d(x2, self.ndim)
        v = np.asarray(v, dtype=np.float64)
        n1, n2 = x1.shape[0], x2.shape[0]
        if v.shape == (n2,):
            v, ldv = np.ascontiguousarray(v), 0
        elif v.shape == (n2, n1):
            v, ldv = np.asfortranarray(v), n2
        else:
            raise DimensionMismatch("dimension mismatch")
        out = np.empty((n1, self.ndim), dtype=np.float64)
        _lib.check(_lib.load().bgp_kmat_x1_gradient_matvec(C.byref(self._spec), _lib.ptr(x1), n1, _lib.ptr(x2), n2,
                                                           _lib.ptr(v), ldv, float(scale), 1 if add_prior else 0,
                                                           _lib.ptr(out)))
        return out

    def _x_gradient(self, fn, x1, x2):
        x1, x2 = _as2d(x1, self.ndim), _as2d(x2, self.ndim)
        out = np.empty((x1.shape[0], x2.shape[0], self.ndim), dtype=np.float64)
        _lib.check(fn(C.byref(self._spec), _lib.ptr(x1), x1.shape[0], _lib.ptr(x2), x2.shape[0], _lib.ptr(out)))
        return out

    def x1_gradient_general(self, x1, x2):
        """d k(x1_i, x2_j) / d x1_i, shape (n1, n2, ndim) (reference kernel_interface.cpp:127-141)."""
        return self._x_gradient(_lib.load().bgp_kmat_x1_gradient_general, x1, x2)

    def x2_gradient_general(self, x1, x2):
        """d k(x1_i, x2_j) / d x2_j, shape (n1, n2, ndim) (reference kernel_interface.cpp:143-157)."""
        return self._x_gradient(_lib.load().bgp_kmat_x2_gradient_general, x1, x2)
