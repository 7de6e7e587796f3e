# -*- coding: utf-8 -*-
"""The HODLR symmetric factor K~ = W W^T on a sharded factorisation (DESIGN.md §5), on ONE device through the
host-exchange entry points of ``include/bgp.h``: P handles finished as in ``test_gpu_hodlr_shards.py``, then
``bgp_hodlr_sym_factor_local`` on every shard, ``sym_export_top`` into one (P, cols, rows_pad) device buffer,
``sym_import_top`` and ``sym_finish_top`` on every shard.  W z is ``sym_apply_top_dev`` then ``sym_apply_local_dev`` on
every shard and the host assembling shard s's rows; W^T z is local, the host's assembly, then top.  That runs every
sharded address and kernel of a P-GPU build and apply; only the all-gather's transport differs from the NCCL path.

The references are an unsharded ``rng_mode="pernode"`` handle on the same problem (the same ranks, pivots and factors,
``test_gpu_hodlr_shards.py``) and K~ assembled from its factors as ``test_gpu_hodlr_sqrt.py`` does.
"""

import ctypes as C

import numpy as np
import pytest

import test_gpu_hodlr_shards as hs
import test_gpu_hodlr_sqrt as sq

pytestmark = pytest.mark.gpu

# bars: 10-100x the largest value measured on one H100 80GB HBM3 (SXM, 700 W power limit) over the cases here.  The
# sharded W(I) agreed with the unsharded handle's bit for bit in every case (each product sums in a fixed order per node
# and column, whichever part of the panel holds a level), so its bar is a rounding-level floor, not a multiple.
TOL_W = 1e-14        # max |W_sharded(I) - W_single(I)| / max |W_single|                      (measured 0)
TOL_TRANS = 1e-13    # max |W^T_sharded(I) - W_sharded(I)^T| / max |W|                         (measured 2.7e-15)
TOL_FACTOR = 1e-13   # max |W W^T - K~| / max |K~|, K~ from the unsharded handle's factors      (measured 6.2e-15)
TOL_LOGDET = 1e-13   # |sum of the partial log|K~| - reference| / max(1, |reference|)          (measured 5.5e-15)
TOL_WHITEN = 1e-13   # max |(W Z)^T K~^-1 (W Z) - Z^T Z| / max |Z^T Z|, N = 2^17, P = 4         (measured 9.9e-16)

NRHS = [1, 63, 64, 65, 130]
BGP_OK, BGP_ERR_INVALID, BGP_ERR_NOT_COMPUTED = 0, 1, 3

# test_gpu_hodlr_shards.py's cases small enough for dense references (n <= ~2048), P = 2, 4 and 8
SMALL = [c for c in hs.CASES if c[1] <= 2048]


def _lib():
    from george_b200 import _lib
    return _lib


def _sym_exchange(sh):
    """The symmetric factor on every shard of ``sh``: factor_local, then _sym_finish.  Returns the partial log|K~| of
    every shard."""
    for s in sh.handles:
        s.symmetric_factor_local()
    return _sym_finish(sh)


def _sym_finish(sh):
    """export_top of every shard into one (P, cols, rows_pad) device buffer, a device synchronise, import_top and
    finish_top on every shard."""
    lib = _lib().load()
    rows_pad = max(rows for _, rows in sh.ranges)
    buf = hs._Dev(sh.P * sh.cols * rows_pad)
    for r, s in enumerate(sh.handles):
        s.symmetric_export_top(buf.at(r * sh.cols * rows_pad), rows_pad)
    _lib().check(lib.bgp_dev_synchronize())
    for s in sh.handles:
        s.symmetric_import_top(buf.p, rows_pad)
    return [s.symmetric_finish_top() for s in sh.handles]


def _blocks(sh, Z):
    """Z replicated into every shard's (N + PAD) x k column-major device block."""
    n, k = Z.shape
    ldz = n + hs.PAD
    blk = np.full((k, ldz), hs.FILL)
    blk[:, :n] = Z.T
    bufs = [hs._Dev(k * ldz) for _ in sh.handles]
    for b in bufs:
        b.upload(blk)
    return bufs, ldz


def _download(bufs, n, k, ldz):
    out = [b.download().reshape(k, ldz) for b in bufs]
    for o in out:
        assert np.all(o[:, n:] == hs.FILL)  # the PAD rows are never written
    return out


def _assemble_rows(sh, blocks, n, k, ldz):
    asm = np.full((k, ldz), hs.FILL)
    for (row0, rows), blk in zip(sh.ranges, blocks):
        asm[:, row0:row0 + rows] = blk[:, row0:row0 + rows]
    return asm


def _sharded_apply(sh, Z, transpose=False):
    """W Z (or W^T Z) on the shards.  Returns (result, tops): ``tops`` are the P shards' blocks after their top part
    (W: before the local part, W^T: the results), which must agree bit for bit."""
    n, k = Z.shape
    bufs, ldz = _blocks(sh, Z)
    if not transpose:
        for s, b in zip(sh.handles, bufs):
            s.apply_symmetric_factor_top(b.p, k, ldz)
        tops = _download(bufs, n, k, ldz)
        for s, b in zip(sh.handles, bufs):
            s.apply_symmetric_factor_local(b.p, k, ldz)
        out = _assemble_rows(sh, _download(bufs, n, k, ldz), n, k, ldz)
        return out[:, :n].T, [t[:, :n].T for t in tops]
    for s, b in zip(sh.handles, bufs):
        s.apply_symmetric_factor_local(b.p, k, ldz, transpose=True)
    asm = _assemble_rows(sh, _download(bufs, n, k, ldz), n, k, ldz)
    for b in bufs:
        b.upload(asm)
    for s, b in zip(sh.handles, bufs):
        s.apply_symmetric_factor_top(b.p, k, ldz, transpose=True)
    tops = [t[:, :n].T for t in _download(bufs, n, k, ldz)]
    return tops[0], tops


def _rel(a, b):
    return float(np.max(np.abs(a - b)) / np.max(np.abs(b)))


# ---- 1. P = 1: local + top are the whole apply ------------------------------------------------------------------------

@pytest.mark.parametrize("transpose", [False, True])
def test_unsharded_local_and_top_give_sym_apply_bits(gpu, transpose):
    kernel, x, yerr, _ = hs._problem("m32", 4097)
    s = hs._single(kernel, x, yerr, min_size=64, tol=1e-10, exhaust="lowrank")
    n = x.shape[0]
    Z = np.random.default_rng(4).standard_normal((n, max(NRHS)))
    sh = hs._Shards([s], [(0, n)], 0, [])
    for k in NRHS:
        want = s.apply_symmetric_factor(Z[:, :k], transpose=transpose)
        got, _ = _sharded_apply(sh, Z[:, :k], transpose)
        assert np.array_equal(got, want), k
    # and the step-by-step build on one handle is the whole factor: the same log|K~| and the same bits
    ld = s.symmetric_log_determinant
    assert _sym_exchange(sh) == [ld]
    assert np.array_equal(_sharded_apply(sh, Z[:, :65], transpose)[0], s.apply_symmetric_factor(Z[:, :65], transpose))


# ---- 2./3./5. against the unsharded handle ---------------------------------------------------------------------------

@pytest.mark.parametrize("case", SMALL, ids=hs._case_id)
def test_sharded_factor_against_unsharded(gpu, record_property, case):
    name, n, min_size, P, exhaust, tol, small = case
    with pytest.MonkeyPatch.context() as mp:
        for var in ("BGP_SMALL_RANK_LIMIT", "BGP_SYM_QR"):
            mp.delenv(var, raising=False)
        if small is not None:
            mp.setenv("BGP_SMALL_RANK_LIMIT", small)
        kernel, x, yerr, _ = hs._problem(name, n)
        opts = dict(min_size=min_size, tol=tol, exhaust=exhaust)
        single = hs._single(kernel, x, yerr, **opts)
        sh = hs._shards(kernel, x, yerr, P, **opts)
        partial = _sym_exchange(sh)
    x2 = x if x.ndim == 2 else x[:, None]
    I = np.eye(n)
    W1 = single.apply_symmetric_factor(I)
    W, tops = _sharded_apply(sh, I)
    Wt, tops_t = _sharded_apply(sh, I, transpose=True)
    for tt in (tops, tops_t):  # the top levels: the same launches on the same data on every shard
        for t in tt[1:]:
            assert np.array_equal(t, tt[0])
    Kt = sq._assemble(single, kernel, x2, yerr)
    errs = {"w": _rel(W, W1), "trans": _rel(Wt, W.T), "factor": _rel(W @ W.T, Kt)}
    ld_single = single.symmetric_log_determinant
    ld_parts = sum(s.log_determinant for s in sh.handles)
    errs["logdet"] = abs(sum(partial) - ld_single) / max(1.0, abs(ld_single))
    errs["logdet_parts"] = abs(sum(partial) - ld_parts) / max(1.0, abs(ld_parts))
    for k, v in errs.items():
        record_property(k, v)
    record_property("bits_equal_unsharded", bool(np.array_equal(W, W1)))
    assert errs["w"] <= TOL_W and errs["trans"] <= TOL_TRANS and errs["factor"] <= TOL_FACTOR, errs
    assert errs["logdet"] <= TOL_LOGDET and errs["logdet_parts"] <= TOL_LOGDET, errs

    # 5. the local part reads and writes only its own rows: NaN elsewhere leaves its rows as they were
    Z = np.random.default_rng(n + P).standard_normal((n, 9))
    for transpose in (False, True):
        bufs, ldz = _blocks(sh, Z)
        for s, b in zip(sh.handles, bufs):
            s.apply_symmetric_factor_local(b.p, 9, ldz, transpose=transpose)
        ref = _download(bufs, n, 9, ldz)
        for r, ((row0, rows), s) in enumerate(zip(sh.ranges, sh.handles)):
            blk = np.full((9, ldz), np.nan)
            blk[:, n:] = hs.FILL
            blk[:, row0:row0 + rows] = Z.T[:, row0:row0 + rows]
            b = hs._Dev(9 * ldz)
            b.upload(blk)
            s.apply_symmetric_factor_local(b.p, 9, ldz, transpose=transpose)
            got = b.download().reshape(9, ldz)
            assert np.array_equal(got[:, row0:row0 + rows], ref[r][:, row0:row0 + rows]), (r, transpose)
            outside = np.ones(ldz, dtype=bool)
            outside[row0:row0 + rows] = False
            outside[n:] = False
            assert np.all(np.isnan(got[:, outside])), (r, transpose)

    # 5. a second build gives the same bits
    assert _sym_exchange(sh) == partial
    assert np.array_equal(_sharded_apply(sh, I)[0], W)


def test_sharded_top_parts_agree_bit_for_bit(gpu):
    """The deepest case at P = 8: every shard's top part of W^T z and of W z is the same array."""
    kernel, x, yerr, _ = hs._problem("m32", 4097)
    sh = hs._shards(kernel, x, yerr, 8, min_size=64, tol=1e-10, exhaust="lowrank")
    _sym_exchange(sh)
    Z = np.random.default_rng(8).standard_normal((4097, 65))
    for transpose in (False, True):
        _, tops = _sharded_apply(sh, Z, transpose)
        for t in tops[1:]:
            assert np.array_equal(t, tops[0]), transpose


# ---- 4. whitening at scale ----------------------------------------------------------------------------------------

def test_whitening_at_scale_on_four_shards(gpu, record_property):
    """(W Z)^T K~^-1 (W Z) = Z^T Z at N = 2^17 on four shards, the solve by the sharded split solve: no dense matrix."""
    from george_b200 import kernels
    n, P = 1 << 17, 4
    x = np.sort(np.random.default_rng(1234).uniform(0, 10 * n / 1000, n))[:, None]
    sh = hs._shards(1.0 * kernels.Matern32Kernel(1.0), x, 0.1 * np.ones(n), P, min_size=256, tol=1e-10,
                    exhaust="lowrank")
    partial = _sym_exchange(sh)
    Z = np.random.default_rng(7).standard_normal((n, 8))
    Y, _ = _sharded_apply(sh, Z)
    G = Y.T @ hs._sharded_solve(sh, Y)[0]
    werr = float(np.max(np.abs(G - Z.T @ Z)) / np.max(np.abs(Z.T @ Z)))
    ld_parts = sum(s.log_determinant for s in sh.handles)
    lerr = abs(sum(partial) - ld_parts) / abs(ld_parts)
    record_property("whiten_err", werr)
    record_property("logdet_rel", lerr)
    record_property("build_ms", [s.symmetric_factor_timing()["build_ms"] for s in sh.handles])
    assert werr <= TOL_WHITEN and lerr <= TOL_LOGDET


# ---- 6. failures ----------------------------------------------------------------------------------------------------

def test_bad_leaf_on_one_shard(gpu):
    """A noise-free, numerically rank-one block on shard 1's rows only (test_gpu_hodlr_sqrt.py's negative pivot): that
    shard's local build raises LinAlgError naming the leaf, its finish is refused, shard 0 builds; the device and both
    handles stay usable."""
    from george_b200 import kernels
    lib = _lib().load()
    n = 200
    x = np.linspace(0, 1, n)[:, None]
    yerr = np.where(np.arange(n) < 100, 1.0, 0.0)
    sh = hs._shards(1.0 * kernels.ExpSquaredKernel(1e8), x, yerr, 2, min_size=64, tol=1e-12)
    assert sh.ranges == [(0, 100), (100, 100)]
    sh.handles[0].symmetric_factor_local()
    with pytest.raises(np.linalg.LinAlgError, match=r"not positive definite: leaf 0 \(rows \[100, 200\)\)"):
        sh.handles[1].symmetric_factor_local()
    out = C.c_double()
    assert lib.bgp_hodlr_sym_finish_top(sh.handles[1]._ptr, C.byref(out)) == BGP_ERR_NOT_COMPUTED
    assert "failed" in _lib().last_error()
    buf = hs._Dev(2 * max(sh.cols, 1) * 100)
    assert lib.bgp_hodlr_sym_export_top(sh.handles[1]._ptr, buf.p, 100) == BGP_ERR_NOT_COMPUTED
    # the device and the handles stay usable: the solves still run, and a good problem builds on the same handles
    B = np.random.default_rng(1).normal(size=(n, 3))
    hs._sharded_solve(sh, B)
    kernel, x, yerr, _ = hs._problem("exp", 1024)
    good = hs._shards(kernel, x, yerr, 2, handles={0: sh.handles[0], 1: sh.handles[1]}, min_size=32, tol=1e-12)
    ld = good.log_determinant
    assert abs(sum(_sym_exchange(good)) - ld) <= TOL_LOGDET * abs(ld)


def test_rank_above_the_limit_is_rejected_before_any_launch(gpu):
    """A top node of rank 2049 (above the symmetric factor's 2048): factor_local raises ValueError naming it and
    launches nothing; the solver's factorisation is untouched."""
    import test_gpu_hodlr_sym_blocks as sb
    from george_b200 import kernels
    from ou_reference import exp_problem
    lib = _lib().load()
    n = 2 * (sb.SY_MAX_RANK + 1)
    x = exp_problem(n, 1.0, seed=n)[:, None]
    sh = hs._shards(1.0 * kernels.ExpKernel(1.0), x, np.zeros(n), 2, min_size=sb.SY_MAX_RANK + 1, tol=1e-12)
    assert sh.handles[0].nodes()[0]["rank"] == sb.SY_MAX_RANK + 1
    ld = [s.log_determinant for s in sh.handles]
    msg = r"node 0 \(rows \[0, {0}\), level 0\) has rank {1}, above the symmetric factor's limit of {2}".format(
        n, sb.SY_MAX_RANK + 1, sb.SY_MAX_RANK)
    for s in sh.handles:
        before = lib.bgp_launch_count()
        with pytest.raises(ValueError, match=msg):
            s.symmetric_factor_local()
        assert lib.bgp_launch_count() == before
        assert lib.bgp_hodlr_sym_finish_top(s._ptr, None) == BGP_ERR_NOT_COMPUTED
    assert [s.log_determinant for s in sh.handles] == ld


def test_call_order_errors(gpu):
    lib = _lib().load()
    out = C.c_double()
    fresh = hs._native()
    assert lib.bgp_hodlr_sym_factor_local(fresh._ptr) == BGP_ERR_NOT_COMPUTED  # before compute
    kernel, x, yerr, _ = hs._problem("exp", 1001)
    opts = dict(min_size=60, tol=1e-12)
    pending = hs._native()
    _lib().check(hs._compute_status(pending, kernel, x, yerr, shard_rank=1, shard_count=2, **opts))
    assert lib.bgp_hodlr_sym_factor_local(pending._ptr) == BGP_ERR_NOT_COMPUTED  # before the solver's finish_top

    sh = hs._shards(kernel, x, yerr, 2, **opts)
    assert sh.ranges == [(0, 500), (500, 501)]
    s0, s1 = sh.handles
    buf = hs._Dev(2 * sh.cols * 501)
    z = hs._Dev(1001)
    z.upload(np.ones(1001))
    # before factor_local: export, import, finish and the applies
    assert lib.bgp_hodlr_sym_export_top(s0._ptr, buf.p, 501) == BGP_ERR_NOT_COMPUTED
    assert lib.bgp_hodlr_sym_import_top(s0._ptr, buf.p, 501) == BGP_ERR_NOT_COMPUTED
    assert lib.bgp_hodlr_sym_finish_top(s0._ptr, C.byref(out)) == BGP_ERR_NOT_COMPUTED
    assert lib.bgp_hodlr_sym_apply_local_dev(s0._ptr, z.p, 1, 1001, 0) == BGP_ERR_NOT_COMPUTED
    assert lib.bgp_hodlr_sym_apply_top_dev(s0._ptr, z.p, 1, 1001, 0) == BGP_ERR_NOT_COMPUTED
    # the full entries stay rejected on a host-exchange shard
    assert lib.bgp_hodlr_sym_factor(s0._ptr) == BGP_ERR_INVALID and "sharded" in _lib().last_error()
    for s in sh.handles:
        s.symmetric_factor_local()
    # after factor_local, before finish: the applies; a short rows_pad
    assert lib.bgp_hodlr_sym_apply_local_dev(s0._ptr, z.p, 1, 1001, 1) == BGP_ERR_NOT_COMPUTED
    assert lib.bgp_hodlr_sym_export_top(s1._ptr, buf.p, 500) == BGP_ERR_INVALID  # 501 rows of its own
    _lib().check(lib.bgp_hodlr_sym_export_top(s0._ptr, buf.p, 500))
    assert lib.bgp_hodlr_sym_import_top(s0._ptr, buf.p, 500) == BGP_ERR_INVALID  # shard 1 has 501
    launches = lib.bgp_launch_count()
    assert lib.bgp_hodlr_sym_import_top(s1._ptr, buf.p, 500) == BGP_ERR_INVALID
    assert lib.bgp_launch_count() == launches
    # the rejected calls left the exchange open: it completes as a fresh pair's does
    partial = _sym_finish(sh)
    ref = hs._shards(kernel, x, yerr, 2, **opts)
    assert partial == _sym_exchange(ref)
    # a second finish, and export / import after it
    for s in sh.handles:
        assert lib.bgp_hodlr_sym_finish_top(s._ptr, C.byref(out)) == BGP_ERR_INVALID
        assert lib.bgp_hodlr_sym_export_top(s._ptr, buf.p, 501) == BGP_ERR_INVALID
        assert lib.bgp_hodlr_sym_import_top(s._ptr, buf.p, 501) == BGP_ERR_INVALID
    Z = np.random.default_rng(3).standard_normal((1001, 5))
    assert np.array_equal(_sharded_apply(sh, Z)[0], _sharded_apply(ref, Z)[0])
    # a new compute makes the factor stale again
    _lib().check(hs._compute_status(s0, kernel, x, yerr, shard_rank=0, shard_count=2, **opts))
    assert lib.bgp_hodlr_sym_export_top(s0._ptr, buf.p, 501) == BGP_ERR_NOT_COMPUTED

