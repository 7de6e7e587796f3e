# -*- coding: utf-8 -*-
"""
Host-side helpers around the GP object (sampling, sample ordering, gradient checks).  Outside the accelerated
path; same public functions as the reference's ``src/george/utils.py:11-92``.
"""

import numpy as np
from scipy.spatial import cKDTree

from . import _lib

__all__ = ["multivariate_gaussian_samples", "device_gaussian_samples", "nd_sort_samples", "check_gradient"]


def multivariate_gaussian_samples(matrix, N, mean=None):
    """Draw ``N`` samples from N(mean, matrix); returns shape ``(N, dim)`` or ``(dim,)`` when ``N == 1``."""
    matrix = np.asarray(matrix)
    if mean is None:
        mean = np.zeros(len(matrix))
    draws = np.random.multivariate_normal(mean, matrix, N)
    return draws[0] if N == 1 else draws


def device_gaussian_samples(matrix, z, mean, jitter):
    """``mean + z @ L.T`` (shape ``(size, ns)``) with ``L`` the lower Cholesky factor of ``sym(matrix) + jitter * I``,
    computed on the device (``include/bgp.h: bgp_mvn_sample``).  ``sym`` mirrors the lower triangle of ``matrix``
    (``(ns, ns)``); ``z`` (``(size, ns)``) holds the caller's standard normals, so the draws are reproducible from
    them.  Raises ``numpy.linalg.LinAlgError`` when that matrix is not positive definite, where
    :func:`multivariate_gaussian_samples` warns and draws anyway."""
    matrix = np.ascontiguousarray(matrix, dtype=np.float64)
    z = np.ascontiguousarray(z, dtype=np.float64)
    mean = np.ascontiguousarray(mean, dtype=np.float64)
    ns = len(mean)
    if matrix.shape != (ns, ns) or z.ndim != 2 or z.shape[1] != ns:
        raise ValueError("matrix must be (ns, ns) and z (size, ns) for a mean of length ns")
    out = np.empty(z.shape, dtype=np.float64)
    _lib.check(_lib.load().bgp_mvn_sample(_lib.ptr(matrix), ns, _lib.ptr(mean), _lib.ptr(z), z.shape[0],
                                          float(jitter), _lib.ptr(out)))
    return out


def nd_sort_samples(samples):
    """Indices that order ``(nsamples, ndim)`` points along a nearest-neighbour walk from the origin-most point,
    which keeps the off-diagonal blocks of a kernel matrix low-rank for the HODLR solver."""
    samples = np.asarray(samples)
    assert samples.ndim == 2
    tree = cKDTree(samples)
    _, order = tree.query(np.zeros(samples.shape[1]), k=len(samples))
    return order


def check_gradient(obj, *args, **kwargs):
    """Compare ``obj.get_gradient`` with centred finite differences of ``obj.get_value``."""
    eps = kwargs.pop("eps", 1.23e-5)
    analytic = obj.get_gradient(*args, **kwargs)
    p = obj.get_parameter_vector()
    for i, pi in enumerate(p):
        p[i] = pi + eps
        obj.set_parameter_vector(p)
        plus = obj.get_value(*args, **kwargs)
        p[i] = pi - eps
        obj.set_parameter_vector(p)
        minus = obj.get_value(*args, **kwargs)
        p[i] = pi
        obj.set_parameter_vector(p)
        fd = 0.5 * (plus - minus) / eps
        assert np.allclose(analytic[i], fd), "grad computation failed for '{0}' ({1})".format(
            obj.get_parameter_names()[i], i)
