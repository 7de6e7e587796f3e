# -*- coding: utf-8 -*-
"""``GP.grad_log_likelihood_x`` on the headline workload at full size: cfg3 (Matern-3/2 1-D, leaf 256, tol 1e-10) at
N = 2^18 on the streamed HODLR path, where no dense reference exists, and four host-exchange shards at N = 2^17 against
the unsharded handle.

* translation invariance, exact for a stationary kernel with a constant mean: ``|sum_i dx_i|`` at rounding level
  relative to ``sum_i |dx_i|``;
* ``grad`` is ``grad_log_likelihood``'s to rounding: at this size the HODLR solve sums with atomics (bit-reproducible
  only up to N = 1024), so two ``grad_log_likelihood`` calls differ in their last bits as well;
* the four shards' assembled ``dx`` (``bgp_hodlr_grad_x_terms_local_dev``) against the unsharded streamed entry.
"""
import numpy as np
import pytest

import test_gpu_hodlr_shards as sh
from test_gpu_grad_x import _dev_of

pytestmark = pytest.mark.gpu

SHIFT_TOL = 1e-12  # |sum dx| / sum |dx|                                      (measured 1.7e-15 at N = 700)
SHARD_TOL = 1e-12  # assembled shards vs the unsharded handle, relative to max |dx|   (measured 1.1e-14)
GRAD_TOL = 1e-12   # grad vs grad_log_likelihood, per entry, relative
SENTINEL = -321.5


def _bench_data(n):  # bench.py's inputs
    rng = np.random.default_rng(1234)
    x = np.sort(rng.uniform(0, 10 * n / 1000, n))
    yerr = 0.1 * np.ones(n)
    y = np.sin(x) + 0.1 * rng.normal(size=n)
    return x, yerr, y


@pytest.fixture
def clean(monkeypatch):
    from george_b200.solvers._hodlr import HODLRSolver
    monkeypatch.delenv("BGP_GRAD_CHUNK", raising=False)
    HODLRSolver.release_parked()
    yield
    HODLRSolver.release_parked()


def test_cfg3_full_size(gpu, clean, record_property):
    import george_b200 as george
    from george_b200 import kernels
    from george_b200.solvers import HODLRSolver
    x, yerr, y = _bench_data(1 << 18)
    gp = george.GP(1.0 * kernels.Matern32Kernel(1.0), solver=HODLRSolver, min_size=256, tol=1e-10, exhaust="lowrank")
    gp.compute(x, yerr)
    grad, dx = gp.grad_log_likelihood_x(y, return_gradient=True)
    assert gp.solver.solver.grad_timing()["slabs"] > 0  # streamed
    ref, again = gp.grad_log_likelihood(y), gp.grad_log_likelihood(y)
    record_property("grad_rel", float(np.max(np.abs(grad - ref) / np.abs(ref))))
    record_property("grad_self_rel", float(np.max(np.abs(again - ref) / np.abs(ref))))
    assert np.all(np.abs(grad - ref) <= GRAD_TOL * np.abs(ref))
    assert dx.shape == (1 << 18, 1) and np.all(np.isfinite(dx))
    shift = abs(dx.sum()) / np.abs(dx).sum()
    record_property("shift", float(shift))
    assert shift < SHIFT_TOL


def test_four_shards_at_2_17(gpu, clean, record_property):
    from george_b200 import _lib, kernels
    n = 1 << 17
    x, yerr, y = _bench_data(n)
    x = x[:, None]
    kernel = 1.0 * kernels.Matern32Kernel(1.0)
    opts = dict(min_size=256, tol=1e-10, exhaust="lowrank")
    single = sh._single(kernel, x, yerr, **opts)
    which = np.ones(2, dtype=np.uint32)
    alpha, g, diag, dx = np.empty(n), np.zeros(2), np.empty(n), np.empty(n)
    _lib.check(single._lib.bgp_hodlr_grad_x_terms(single._ptr, _lib.ptr(which), _lib.ptr(y), _lib.ptr(alpha),
                                                  _lib.ptr(g), _lib.ptr(diag), _lib.ptr(dx)))
    del single
    shards = sh._shards(kernel, x, yerr, 4, **opts)
    alphas = [o[:, 0].copy() for o in sh._sharded_solve(shards, y[:, None])]
    assembled = np.full(n, np.nan)
    for s, (row0, rows), a in zip(shards.handles, shards.ranges, alphas):
        ad, dd = _dev_of(a, n), _dev_of(np.full(n, SENTINEL), n)
        s.grad_x_terms_local(ad.p, which, dd.p)
        d = dd.download()
        assert np.all(np.r_[d[:row0], d[row0 + rows:]] == SENTINEL)
        assembled[row0:row0 + rows] = d[row0:row0 + rows]
    rel = float(np.max(np.abs(assembled - dx)) / np.max(np.abs(dx)))
    record_property("rel", rel)
    assert rel < SHARD_TOL
