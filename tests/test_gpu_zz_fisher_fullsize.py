# -*- coding: utf-8 -*-
"""``GP.fisher_information`` on the dense solver at N = 16384: the headline Matern-3/2 1-D inputs of bench.py with a
fitted amplitude, scale and white noise (``yerr = 0``, the noise all in the white-noise model, so that
``dK_c + dK_w = K``):

* the scale identity: the sum of ``F``'s (log c, white noise) block is N / 2;
* exact symmetry, positive semi-definiteness and two calls bit-identical;
* ``grad`` from ``fisher_information(y)`` is ``grad_log_likelihood(y)``'s bits.

The call time is recorded as ``fisher_s`` (and ``grad_s`` for ``grad_log_likelihood``).
"""
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N = 16384
SCALE_TOL = 1e-10  # sum of the (log c, white noise) block vs N / 2, relative
PSD_TOL = 1e-12    # min eigenvalue >= -PSD_TOL * ||F||


def test_headline_dense_fisher(gpu, record_property):
    import george_b200 as george
    from george_b200 import kernels
    rng = np.random.default_rng(1234)  # bench.py's inputs
    x = np.sort(rng.uniform(0, 10 * N / 1000, N))
    y = np.sin(x) + 0.1 * rng.normal(size=N)
    gp = george.GP(1.0 * kernels.Matern32Kernel(1.0), white_noise=np.log(0.1 ** 2), fit_white_noise=True)
    gp.compute(x, 0.0)
    assert gp.get_parameter_names() == ("white_noise:value", "kernel:k1:log_constant", "kernel:k2:metric:log_M_0_0")
    t0 = time.perf_counter()
    grad, F = gp.fisher_information(y)
    record_property("fisher_s", time.perf_counter() - t0)
    t0 = time.perf_counter()
    ref = gp.grad_log_likelihood(y)
    record_property("grad_s", time.perf_counter() - t0)
    assert np.array_equal(grad, ref)
    block = F[:2, :2].sum()
    err = abs(block - N / 2) / (N / 2)
    record_property("scale_rel_err", err)
    assert err < SCALE_TOL, (block, N / 2)
    assert np.array_equal(F, F.T)
    w = np.linalg.eigvalsh(F)
    record_property("min_eig_rel", float(w[0] / np.abs(w).max()))
    assert w[0] >= -PSD_TOL * np.abs(w).max(), w
    assert np.array_equal(F, gp.fisher_information())
