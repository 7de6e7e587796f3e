# -*- coding: utf-8 -*-
"""The sharded HODLR factorisation and solve (``opts.shard_count > 1``, DESIGN.md §5) on ONE device, through the
host-exchange entry points of ``include/bgp.h``.

One process holds P handles on the same GPU, computes handle r with ``shard_rank = r, shard_count = P`` and runs the
all-gather itself: ``export_top`` into a (P, cols, rows_pad) device buffer, ``import_top`` and ``finish_top`` on every
shard; a solve is ``solve_local_dev`` on every shard, the host assembles shard s's rows, ``solve_top_dev`` on every
shard.  That runs every sharded kernel and panel-set address a P-GPU run does (the owned levels' nloc-row panels behind
``PanelSet::vbase()``, the sub-tree pass over this shard's rows of the top panel, pack / unpack, the top nodes and the
partial log-determinants); only the transport differs from the NCCL path.

References: the per-node RNG streams do not depend on the sharding, so an unsharded ``rng_mode="pernode"`` handle on the
same problem fixes the structure exactly (ranks, draws, dense fallbacks, pivots) and the numbers to rounding; on the
exact-K problems of ``test_gpu_hodlr_sweeps.py`` (sorted 1-D ``ExpKernel``, ``exhaust="dense"``: the HODLR matrix IS K)
the numbers are also compared with a longdouble factorisation of K, at that file's bars.
"""

import ctypes as C

import numpy as np
import pytest

import test_gpu_hodlr_sweeps as sw

pytestmark = pytest.mark.gpu

LD = np.longdouble

# bars: sharded vs the unsharded handle on the same device, at most 100x the largest value measured on one H100 80GB
# HBM3 (SXM, 700 W power limit) over all CASES.  The two orders of work differ (the top panel's columns get the sub-tree
# inverse in a pass of their own, the Gram products add their row slices with atomics), so the numbers agree to
# rounding, not bits.  The exact-K cases also meet test_gpu_hodlr_sweeps.py's longdouble bars (measured: log-det
# 5.7e-15, solves 3.2e-13, residuals 2.0e-16).
LOGDET_TOL = 5e-14      # |sum of the P partial log-dets - single| / max(1, |single|)       (measured 6.4e-16)
SOLVE_TOL = 1e-11       # ||X_sharded - X_single|| / ||X_single||                           (measured 1.4e-13)
SPREAD_TOL = 1e-11      # shard r's solve vs shard 0's where the top sums are not order-free (measured 2.1e-13)
DOT_TOL = 2e-13         # y^T K^-1 y from the sharded solve vs the single handle's dot_solve (measured 5.2e-15)
REUSE_TOL = sw.REUSE_TOL  # a reused handle vs a fresh one (measured 0 here, 1.3e-16 in test_gpu_hodlr_sweeps.py)

NRHS = [1, 63, 64, 65, 130]  # the 64-column batches of hodlr_solve_dev and a ragged tail
PAD = 3                      # rows below N in every device right-hand side block (ldb = N + 3): never written
FILL = 7.0

BGP_OK, BGP_ERR_INVALID, BGP_ERR_NOT_COMPUTED, BGP_ERR_RANK_CAPACITY, BGP_ERR_INDEX = 0, 1, 3, 7, 8


def _lib():
    from george_b200 import _lib
    return _lib


@pytest.fixture
def clean(monkeypatch):
    """No diagnostic switch from the environment, and no parked handle left from another test (_native() below also
    releases the parked handles before it creates one)."""
    from george_b200.solvers._hodlr import HODLRSolver
    for var in ("BGP_SMALL_RANK_LIMIT", "BGP_LEAF_COLS", "BGP_NO_GRAPH", "BGP_NO_CULL", "BGP_LEAF_FACTOR"):
        monkeypatch.delenv(var, raising=False)
    HODLRSolver.release_parked()
    yield monkeypatch
    HODLRSolver.release_parked()


class _Dev(object):
    """float64 device buffer from the library's allocator."""

    def __init__(self, count):
        self.lib = _lib().load()
        self.count = int(count)
        self.p = C.c_void_p()
        _lib().check(self.lib.bgp_dev_alloc(C.byref(self.p), 8 * max(self.count, 1)))

    def at(self, offset):
        return C.c_void_p(self.p.value + 8 * int(offset))

    def upload(self, a):
        a = np.ascontiguousarray(a, dtype=np.float64)
        assert a.size == self.count
        _lib().check(self.lib.bgp_dev_upload(self.p, _lib().ptr(a), a.nbytes))

    def download(self):
        out = np.empty(self.count, dtype=np.float64)
        if self.count:
            _lib().check(self.lib.bgp_dev_download(_lib().ptr(out), self.p, out.nbytes))
        return out

    def __del__(self):
        if self.p:
            self.lib.bgp_dev_free(self.p)
            self.p = C.c_void_p()


def _native():
    """A HODLRSolver on a newly created native handle.  HODLRSolver() would otherwise pick up a handle parked by a solver
    that just died, with that solver's last factorisation in it, and a reference built on it would not be independent
    of the handle-reuse path under test."""
    from george_b200.solvers._hodlr import HODLRSolver
    HODLRSolver.release_parked()
    return HODLRSolver()


def _compute_status(s, kernel, x, yerr, min_size, tol, exhaust="dense", rng_mode="pernode", shard_rank=0,
                    shard_count=1, rank_capacity=0):
    """``bgp_hodlr_compute`` on ``s``'s handle, returning the status code instead of raising."""
    from george_b200._spec import flatten
    x = np.ascontiguousarray(x, dtype=np.float64)
    yerr = np.ascontiguousarray(yerr, dtype=np.float64)
    o = s._opts(min_size, tol, 42, rng_mode, rank_capacity, shard_rank, shard_count, exhaust)
    spec = flatten(kernel)
    s._n, s.shard_count, s._fresh = x.shape[0], int(shard_count), False
    return s._lib.bgp_hodlr_compute(s._ptr, C.byref(spec), _lib().ptr(x), x.shape[0], x.shape[1], _lib().ptr(yerr),
                                    C.byref(o))


def _top_panel(s, download=True):
    """(row0, rows, cols, ld, panel): this shard's row range and a host copy of its (N x cols) top panel."""
    p = C.c_void_p()
    row0, rows, cols, ld = C.c_int64(), C.c_int64(), C.c_int64(), C.c_int64()
    _lib().check(s._lib.bgp_hodlr_top_panel(s._ptr, C.byref(p), C.byref(row0), C.byref(rows), C.byref(cols),
                                            C.byref(ld)))
    panel = np.empty((cols.value, ld.value) if download else (0, 0), dtype=np.float64)
    if panel.size:
        _lib().check(s._lib.bgp_dev_download(_lib().ptr(panel), p, panel.nbytes))
    return row0.value, rows.value, cols.value, ld.value, panel.T


def _shard_rows(s, P):
    out = []
    for r in range(P):
        row0, rows = C.c_int64(), C.c_int64()
        _lib().check(s._lib.bgp_hodlr_shard_rows(s._ptr, r, C.byref(row0), C.byref(rows)))
        out.append((row0.value, rows.value))
    return out


class _Shards(object):
    """P host-exchange shards of one problem, factored and finished."""

    def __init__(self, handles, ranges, cols, panels):
        self.handles, self.ranges, self.cols, self.panels = handles, ranges, cols, panels
        self.P = len(handles)

    @property
    def log_determinant(self):
        return sum(s.log_determinant for s in self.handles)


def _shards(kernel, x, yerr, P, handles=None, **opts):
    """Compute all P shards, then the host's exchange (_exchange)."""
    lib = _lib().load()
    handles = dict(handles or {})
    hs = []
    for r in range(P):
        s = handles.get(r) or _native()
        _lib().check(_compute_status(s, kernel, x, yerr, shard_rank=r, shard_count=P, **opts))
        assert not lib.bgp_hodlr_computed(s._ptr)  # waits for its top levels
        hs.append(s)
    return _exchange(hs)


def _exchange(hs):
    """export_top of every shard into one (P, cols, rows_pad) device buffer, a device synchronise (every handle runs
    on its own streams), import_top and finish_top on every shard."""
    lib = _lib().load()
    P = len(hs)
    ranges = _shard_rows(hs[0], P)
    for s in hs[1:]:
        assert _shard_rows(s, P) == ranges
    rows_pad = max(rows for _, rows in ranges)
    cols = [_top_panel(s, False)[2] for s in hs]
    assert len(set(cols)) == 1, cols
    cols = cols[0]
    buf = _Dev(P * cols * rows_pad)
    for r, s in enumerate(hs):
        row0, rows = _top_panel(s, False)[:2]
        assert (row0, rows) == ranges[r]
        _lib().check(lib.bgp_hodlr_export_top(s._ptr, buf.at(r * cols * rows_pad), rows_pad))
    _lib().check(lib.bgp_dev_synchronize())
    for s in hs:
        _lib().check(lib.bgp_hodlr_import_top(s._ptr, buf.p, rows_pad))
    panels = [_top_panel(s)[4] for s in hs]
    for s in hs:
        _lib().check(lib.bgp_hodlr_finish_top(s._ptr))
        assert lib.bgp_hodlr_computed(s._ptr)
    return _Shards(hs, ranges, cols, panels)


def _sharded_solve(sh, B):
    """K^-1 B on the shards: B replicated into every shard's (N + PAD) x nrhs column-major device block,
    solve_local_dev on each, rows [row0_s, row0_s + rows_s) of shard s assembled on the host and copied to every
    shard, solve_top_dev on each.  Returns the P results; the PAD rows must come back untouched."""
    lib = _lib().load()
    n, nrhs = B.shape
    ldb = n + PAD
    blk = np.full((nrhs, ldb), FILL)  # row-major (nrhs, ldb) = column-major (ldb, nrhs)
    blk[:, :n] = B.T
    bufs = [_Dev(nrhs * ldb) for _ in sh.handles]
    for b in bufs:
        b.upload(blk)
    for s, b in zip(sh.handles, bufs):
        _lib().check(lib.bgp_hodlr_solve_local_dev(s._ptr, b.p, nrhs, ldb))
    local = [b.download().reshape(nrhs, ldb) for b in bufs]
    asm = np.full((nrhs, ldb), FILL)
    for (row0, rows), loc in zip(sh.ranges, local):
        assert np.all(loc[:, n:] == FILL)
        asm[:, row0:row0 + rows] = loc[:, row0:row0 + rows]
    for b in bufs:
        b.upload(asm)
    for s, b in zip(sh.handles, bufs):
        _lib().check(lib.bgp_hodlr_solve_top_dev(s._ptr, b.p, nrhs, ldb))
    out = [b.download().reshape(nrhs, ldb) for b in bufs]
    for o in out:
        assert np.all(o[:, n:] == FILL)
    return [o[:, :n].T for o in out]


def _single(kernel, x, yerr, **opts):
    s = _native()
    _lib().check(_compute_status(s, kernel, x, yerr, **opts))
    return s


def _rel(X, Xr):
    return sw._rel(X, Xr)


# ---- problems ---------------------------------------------------------------------------------------------------

def _problem(name, n):
    """(kernel, x, yerr, longdouble reference or None)."""
    from george_b200 import kernels as K
    if name == "exp":
        return sw._exp_problem(n)
    if name == "clusters":  # test_gpu_hodlr_sweeps.py::test_rank_zero_root_between_two_clusters
        kernel = sw._exp_kernel()
        rng = np.random.default_rng(11)
        x = np.concatenate([np.sort(rng.uniform(0, 4, n // 2)), 104.0 + np.sort(rng.uniform(0, 4, n // 2))])[:, None]
        yerr = 0.1 * np.ones(n)
        return kernel, x, yerr, sw._reference(kernel, x, yerr, ("clusters", n))
    rng = np.random.default_rng(n)
    if name == "m32":
        x, yerr = sw._inputs(n, seed=3)
        return 1.0 * K.Matern32Kernel(1.0), x, yerr, None
    if name == "m52_3d":  # the interpreter: no 1-D shape, no bound culling
        x = rng.uniform(0, 4, (n, 3))
        x = x[np.argsort(x[:, 0])]
        return K.Matern52Kernel(0.5, ndim=3), x, 0.1 * np.ones(n), None
    if name == "cfg5":  # bench config 5's kernel: ExpSine2 has no decay bound
        x = np.sort(rng.uniform(0, 10 * n / 1000, n))[:, None]
        kernel = 1.0 * K.ExpSquaredKernel(1.0) + 0.5 * K.ExpSine2Kernel(gamma=1.0, log_period=np.log(3.0))
        return kernel, x, 0.1 * np.ones(n), None
    raise KeyError(name)


# (problem, N, min_size, P, exhaust, tol, BGP_SMALL_RANK_LIMIT)
CASES = [
    ("exp", 1024, 32, 2, "dense", 1e-12, None),   # even split; root 2r = 1024: DMMA Gram and blocked LU on the top
    ("exp", 1024, 32, 4, "dense", 1e-12, None),   # two top levels (r = 512, 256), the default capacity 128 regrown
    ("exp", 1024, 32, 8, "dense", 1e-12, None),
    ("exp", 1001, 60, 2, "dense", 1e-12, None),   # odd N: 500 / 501 rows, rows_pad pads
    ("exp", 1001, 60, 8, "dense", 1e-12, None),   # 125 / 126-row sub-trees of one internal node each
    ("exp", 799, 100, 4, "dense", 1e-12, None),   # shard 0 owns one 199-row leaf at the cut, the others two leaves
    ("exp", 1001, 60, 4, "dense", 1e-12, "0"),    # every level through launch_level_big
    ("clusters", 400, 50, 2, "lowrank", 1e-12, None),  # rank-0 root: the top panel has no columns
    ("m32", 4097, 64, 2, "lowrank", 1e-10, None),  # deeper tree (7 levels), bound culling, rejection-heavy ACA
    ("m32", 4097, 64, 4, "lowrank", 1e-10, None),
    ("m32", 4097, 64, 8, "lowrank", 1e-10, None),
    ("m52_3d", 1200, 75, 4, "dense", 1e-8, None),
    ("cfg5", 3000, 100, 2, "lowrank", 1e-10, None),
    ("cfg5", 3000, 100, 8, "lowrank", 1e-10, None),
]


def _case_id(c):
    return "{0}-{1}-ms{2}-P{3}{4}".format(c[0], c[1], c[2], c[3], "-smallrank" + c[6] if c[6] is not None else "")


def _factored(nd, cut, row0, rows):
    """An internal node shard [row0, row0 + rows) factors: above the cut, or inside its sub-tree."""
    return nd["depth"] < cut or (row0 <= nd["start"] and nd["start"] + nd["size"] <= row0 + rows)


def _check_structure(sh, single, n, min_size):
    """Check 1: every node a shard factored has the single handle's rank, draws, fallback and pivots; the others
    report rank 0; the shard row ranges are george_b200.parallel.shard_ranges.  Returns the number of nodes compared."""
    from george_b200.parallel import shard_ranges
    assert sh.ranges == [tuple(r) for r in shard_ranges(n, sh.P, min_size)]
    ref = single.nodes()
    geo = ("start", "size", "half", "is_leaf", "parent", "direction", "depth")
    cut = sh.P.bit_length() - 1
    compared = 0
    for s, (row0, rows) in zip(sh.handles, sh.ranges):
        nodes = s.nodes()
        assert [[d[k] for k in geo] for d in nodes] == [[d[k] for k in geo] for d in ref]
        for i, (a, b) in enumerate(zip(nodes, ref)):
            if a["is_leaf"]:
                continue
            if not _factored(a, cut, row0, rows):
                assert a["rank"] == 0 and a["rng_draws"] == 0, (i, a)
                continue
            assert (a["rank"], a["rng_draws"], a["dense_fallback"]) == \
                (b["rank"], b["rng_draws"], b["dense_fallback"]), (i, a, b)
            ra, ca = s.pivots(i, a["rank"])
            rb, cb = single.pivots(i, b["rank"])
            assert np.array_equal(ra, rb) and np.array_equal(ca, cb), i
            compared += 1
    return compared


def _top_sums_are_order_free(single, P, small_limit):
    """Whether every entry of a top level's Gram product W = V^T X is at most two partial sums added into zero with
    atomics (csrc/hodlr.cu: launch_level): 1024-row CTAs for 2r <= 16, 512-row ones up to 2r = 142, 4096-row DMMA
    slices above (or above BGP_SMALL_RANK_LIMIT).  Two addends give the same double in either order, so the P shards'
    top nodes, which run the same launches on the same data, then agree bit for bit; three or more may round
    differently from one launch to the next."""
    cut = P.bit_length() - 1
    nodes = single.nodes()
    for depth in range(cut):
        level = [nd for nd in nodes if not nd["is_leaf"] and nd["depth"] == depth]
        r = max(nd["rank"] for nd in level)
        if r == 0:
            continue
        rows = 4096 if 2 * r > small_limit else 1024 if r <= 8 else 512
        if max(nd["size"] - nd["half"] for nd in level) > 2 * rows:
            return False
    return True


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_sharded_factorisation_and_solve(gpu, clean, record_property, case):
    """Structure, top panel, log-determinant and solves of P host-exchange shards against the unsharded handle (and,
    on the exact-K problems, a longdouble factorisation of K)."""
    name, n, min_size, P, exhaust, tol, small = case
    if small is not None:
        clean.setenv("BGP_SMALL_RANK_LIMIT", small)
    kernel, x, yerr, ref = _problem(name, n)
    opts = dict(min_size=min_size, tol=tol, exhaust=exhaust)
    single = _single(kernel, x, yerr, **opts)
    sh = _shards(kernel, x, yerr, P, **opts)

    # 1. structure
    record_property("nodes_compared", _check_structure(sh, single, n, min_size))
    if name == "exp":
        sw._assert_exact_dense_tree(single, n)
    if name == "clusters":
        assert single.nodes()[0]["rank"] == 0 and sh.cols == 0
    if name == "exp" and n == 1024 and P == 2:
        # The capacity-growth loop with both panel sets (hodlr_compute_dev_impl, "capacities"): the shards above ran on
        # new handles (no capacity hint), so every level started at the automatic capacity, min(128, half); the root
        # (top set, rank 512) and the level below the cut (owned set, rank 256) are above it, so both sets were grown
        # and the ACA rerun.  The same start given as a hard cap is rejected, which pins that it was below the ranks.
        ranks = {nd["depth"]: nd["rank"] for nd in single.nodes() if not nd["is_leaf"]}
        assert ranks[0] > 128 and ranks[1] > 128, ranks
        capped = _native()
        assert _compute_status(capped, kernel, x, yerr, shard_rank=0, shard_count=P, rank_capacity=128,
                               **opts) == BGP_ERR_RANK_CAPACITY

    # 2. after import_top every shard holds the same top panel
    for p in sh.panels[1:]:
        assert p.shape == sh.panels[0].shape and np.array_equal(p, sh.panels[0])

    # 3. the partial log-determinants add up to the single handle's (and K's)
    errs = {"logdet": abs(sh.log_determinant - single.log_determinant) / max(1.0, abs(single.log_determinant))}
    if ref is not None:
        errs["logdet_ld"] = abs(sh.log_determinant - ref.logdet) / max(1.0, abs(ref.logdet))

    # 4. solves
    order_free = _top_sums_are_order_free(single, P, int(small) if small is not None else 142)
    rng = np.random.default_rng(n + P)
    B = ref.B[:, :max(NRHS)] if ref is not None else rng.normal(size=(n, max(NRHS)))
    errs["solve"] = errs["spread"] = errs["solve_ld"] = errs["residual_ld"] = 0.0
    for nrhs in NRHS:
        outs = _sharded_solve(sh, B[:, :nrhs])
        for o in outs[1:]:  # the same assembled input and the same top-level launches on every shard
            if order_free:
                assert np.array_equal(o, outs[0]), nrhs
            errs["spread"] = max(errs["spread"], _rel(o, outs[0]))
        X1 = single.apply_inverse(B[:, :nrhs])
        errs["solve"] = max(errs["solve"], _rel(outs[0], X1))
        if ref is not None:
            errs["solve_ld"] = max(errs["solve_ld"], _rel(outs[0], ref.X[:, :nrhs]))
            if nrhs in (1, 65):  # (O(n^2 nrhs) longdouble)
                errs["residual_ld"] = max(errs["residual_ld"], ref.residual(outs[0], B[:, :nrhs]))
    y = B[:, 0]
    q = float(np.dot(y, _sharded_solve(sh, y[:, None])[0][:, 0]))
    q1 = single.dot_solve(y)
    errs["dot_solve"] = abs(q - q1) / abs(q1)

    for k, v in errs.items():
        record_property(k, v)
    assert errs["logdet"] <= LOGDET_TOL, errs
    assert errs["spread"] <= SPREAD_TOL, errs
    assert errs["solve"] <= SOLVE_TOL and errs["dot_solve"] <= DOT_TOL, errs
    if ref is not None:
        assert errs["logdet_ld"] <= sw.LOGDET_TOL, errs
        assert errs["solve_ld"] <= sw.SOLVE_TOL and errs["residual_ld"] <= sw.RESIDUAL_TOL, errs


def _snapshot(sh, B):
    """Everything a sharded factorisation answers: per shard nodes and pivots, partial log-dets, top panels, solves."""
    out = []
    for s in sh.handles:
        nodes = s.nodes()
        piv = [s.pivots(i, nd["rank"]) for i, nd in enumerate(nodes) if not nd["is_leaf"]]
        out.append((nodes, piv, s.log_determinant))
    return out, sh.panels, _sharded_solve(sh, B)


def _assert_same(a, b, what):
    (sa, pa, Xa), (sb, pb, Xb) = a, b
    worst = 0.0
    for (na, piva, la), (nb, pivb, lb) in zip(sa, sb):
        assert na == nb, what
        for (ra, ca), (rb, cb) in zip(piva, pivb):
            assert np.array_equal(ra, rb) and np.array_equal(ca, cb), what
        worst = max(worst, abs(la - lb) / max(1.0, abs(lb)))
    for p, q in zip(pa, pb):
        worst = max(worst, _rel(p, q) if q.size else 0.0)
    for x, y in zip(Xa, Xb):
        worst = max(worst, _rel(x, y))
    assert worst <= REUSE_TOL, (what, worst)
    return worst


def test_handle_reuse_across_shardings(gpu, clean, record_property):
    """One handle is shard 1 of 4, then shard 0 of 2 at another N, then unsharded: each result equals a fresh
    handle's (structure exactly, numbers to the Gram products' atomic-add noise), and after the unsharded compute
    bgp_hodlr_shard_rows reports no ranges."""
    lib = _lib().load()
    kernel_a, xa, ea, _ = _problem("m32", 4097)
    kernel_b, xb, eb, _ = _problem("exp", 1001)
    opts_a = dict(min_size=64, tol=1e-10, exhaust="lowrank")
    opts_b = dict(min_size=60, tol=1e-12, exhaust="dense")
    rng = np.random.default_rng(5)
    reused = _native()
    worst = 0.0
    # every reference below (`want`, `fresh`) is built on newly created handles (_native), never on one parked by the
    # previous step's solvers

    Ba = rng.normal(size=(4097, 65))
    got = _snapshot(_shards(kernel_a, xa, ea, 4, handles={1: reused}, **opts_a), Ba)
    want = _snapshot(_shards(kernel_a, xa, ea, 4, **opts_a), Ba)
    worst = max(worst, _assert_same(got, want, "shard 1 of 4"))

    Bb = rng.normal(size=(1001, 65))
    got = _snapshot(_shards(kernel_b, xb, eb, 2, handles={0: reused}, **opts_b), Bb)
    want = _snapshot(_shards(kernel_b, xb, eb, 2, **opts_b), Bb)
    worst = max(worst, _assert_same(got, want, "shard 0 of 2"))

    _lib().check(_compute_status(reused, kernel_b, xb, eb, **opts_b))
    fresh = _single(kernel_b, xb, eb, **opts_b)
    assert reused.nodes() == fresh.nodes()
    for i, nd in enumerate(fresh.nodes()):
        if not nd["is_leaf"]:
            ra, ca = reused.pivots(i, nd["rank"])
            rb, cb = fresh.pivots(i, nd["rank"])
            assert np.array_equal(ra, rb) and np.array_equal(ca, cb)
    errs = [abs(reused.log_determinant - fresh.log_determinant) / max(1.0, abs(fresh.log_determinant)),
            _rel(reused.apply_inverse(Bb), fresh.apply_inverse(Bb)),
            abs(reused.dot_solve(Bb[:, 0]) - fresh.dot_solve(Bb[:, 0])) / abs(fresh.dot_solve(Bb[:, 0]))]
    worst = max(worst, max(errs))
    assert max(errs) <= REUSE_TOL, errs
    row0, rows = C.c_int64(), C.c_int64()
    for s in range(2):
        assert lib.bgp_hodlr_shard_rows(reused._ptr, s, C.byref(row0), C.byref(rows)) == BGP_ERR_INDEX
    record_property("reuse_diff", worst)


def test_full_solves_are_rejected_on_a_host_exchange_shard(gpu, clean):
    """apply_inverse, dot_solve[_dev] and get_inverse on a finished host-exchange shard would solve only its own rows
    before the top levels: BGP_ERR_INVALID, naming the split solve, and the shard still solves through it."""
    lib = _lib().load()
    kernel, x, yerr, _ = _problem("exp", 1001)
    sh = _shards(kernel, x, yerr, 2, min_size=60, tol=1e-12)
    B = np.random.default_rng(1).normal(size=(1001, 3))
    before = _sharded_solve(sh, B)
    s = sh.handles[1]
    b = np.asfortranarray(B.copy())
    out = C.c_double()
    assert lib.bgp_hodlr_apply_inverse(s._ptr, _lib().ptr(b), 3, 1001) == BGP_ERR_INVALID
    assert "solve_local_dev" in _lib().last_error() and "solve_top_dev" in _lib().last_error()
    assert np.array_equal(b, B)
    y = np.ascontiguousarray(B[:, 0])
    assert lib.bgp_hodlr_dot_solve(s._ptr, _lib().ptr(y), C.byref(out)) == BGP_ERR_INVALID
    ydev = _Dev(1001)
    ydev.upload(y)
    assert lib.bgp_hodlr_dot_solve_dev(s._ptr, ydev.p, C.byref(out)) == BGP_ERR_INVALID
    inv = np.zeros((1001, 1001))
    assert lib.bgp_hodlr_get_inverse(s._ptr, _lib().ptr(inv)) == BGP_ERR_INVALID
    after = _sharded_solve(sh, B)
    for p, q in zip(before, after):
        assert np.array_equal(p, q)
    # the same handle unsharded answers the full solves again
    _lib().check(_compute_status(s, kernel, x, yerr, min_size=60, tol=1e-12))
    assert _rel(s.apply_inverse(B), before[0]) <= SOLVE_TOL


def test_finish_top_only_once_after_a_sharded_compute(gpu, clean):
    """finish_top: NOT_COMPUTED on a fresh handle, INVALID on an unsharded factorisation and on a second call (the
    first already updated the top panel in place); import_top after it is INVALID too; none of them changes a result."""
    lib = _lib().load()
    s = _native()
    assert lib.bgp_hodlr_finish_top(s._ptr) == BGP_ERR_NOT_COMPUTED
    assert not lib.bgp_hodlr_computed(s._ptr)
    kernel, x, yerr, _ = _problem("exp", 1024)
    opts = dict(min_size=32, tol=1e-12)
    _lib().check(_compute_status(s, kernel, x, yerr, **opts))
    ld = s.log_determinant
    assert lib.bgp_hodlr_finish_top(s._ptr) == BGP_ERR_INVALID
    assert s.log_determinant == ld

    sh = _shards(kernel, x, yerr, 4, handles={0: s}, **opts)
    B = np.random.default_rng(2).normal(size=(1024, 9))
    lds = [h.log_determinant for h in sh.handles]
    before = _sharded_solve(sh, B)
    buf = _Dev(4 * max(sh.cols, 1) * 256)
    for h in sh.handles:
        assert lib.bgp_hodlr_finish_top(h._ptr) == BGP_ERR_INVALID
        assert lib.bgp_hodlr_import_top(h._ptr, buf.p, 256) == BGP_ERR_INVALID
        assert lib.bgp_hodlr_export_top(h._ptr, buf.p, 256) == BGP_ERR_INVALID
    assert [h.log_determinant for h in sh.handles] == lds
    for p, q in zip(before, _sharded_solve(sh, B)):
        assert np.array_equal(p, q)
    assert abs(sh.log_determinant - ld) <= LOGDET_TOL * max(1.0, abs(ld))


def test_import_top_rejects_a_short_rows_pad(gpu, clean):
    """Odd N: shard rows 500 and 501.  rows_pad = 500 is enough for shard 0's export but would make the import read
    shard 1's slice at the wrong offsets: BGP_ERR_INVALID, and an import at 501 afterwards completes the exchange."""
    lib = _lib().load()
    kernel, x, yerr, _ = _problem("exp", 1001)
    opts = dict(min_size=60, tol=1e-12)
    hs = [_native() for _ in range(2)]
    for r, s in enumerate(hs):
        _lib().check(_compute_status(s, kernel, x, yerr, shard_rank=r, shard_count=2, **opts))
    assert _shard_rows(hs[0], 2) == [(0, 500), (500, 501)]
    cols = _top_panel(hs[0], False)[2]
    short = _Dev(2 * cols * 501)  # room for both slices: only the rows_pad argument is short
    _lib().check(lib.bgp_hodlr_export_top(hs[0]._ptr, short.p, 500))
    for s in hs:
        assert lib.bgp_hodlr_import_top(s._ptr, short.p, 500) == BGP_ERR_INVALID
    assert lib.bgp_hodlr_export_top(hs[1]._ptr, short.at(cols * 500), 500) == BGP_ERR_INVALID  # 501 rows of its own
    # the rejected calls left both handles waiting for their exchange: it completes as a fresh pair's does
    sh = _exchange(hs)
    ref = _shards(kernel, x, yerr, 2, **opts)
    for p, q in zip(sh.panels, ref.panels):
        assert _rel(p, q) <= REUSE_TOL
    assert abs(sh.log_determinant - ref.log_determinant) <= REUSE_TOL * abs(ref.log_determinant)
    B = np.random.default_rng(3).normal(size=(1001, 2))
    for p, q in zip(_sharded_solve(sh, B), _sharded_solve(ref, B)):
        assert _rel(p, q) <= REUSE_TOL


def test_split_solve_needs_finish_top(gpu, clean):
    """solve_local_dev / solve_top_dev before finish_top: BGP_ERR_NOT_COMPUTED."""
    lib = _lib().load()
    kernel, x, yerr, _ = _problem("exp", 1024)
    s = _native()
    _lib().check(_compute_status(s, kernel, x, yerr, min_size=32, tol=1e-12, shard_rank=0, shard_count=2))
    b = _Dev(1024)
    b.upload(np.ones(1024))
    assert lib.bgp_hodlr_solve_local_dev(s._ptr, b.p, 1, 1024) == BGP_ERR_NOT_COMPUTED
    assert lib.bgp_hodlr_solve_top_dev(s._ptr, b.p, 1, 1024) == BGP_ERR_NOT_COMPUTED
    out = C.c_double()
    assert lib.bgp_hodlr_log_determinant(s._ptr, C.byref(out)) == BGP_ERR_NOT_COMPUTED


@pytest.mark.parametrize("what,n,min_size,rank,count,rng_mode", [
    ("too_shallow", 300, 100, 0, 4, "pernode"),   # 300 -> 150 | 150, both leaves: no depth-2 node
    ("count_3", 1024, 32, 0, 3, "pernode"),
    ("rank_eq_count", 1024, 32, 4, 4, "pernode"),
    ("rank_negative", 1024, 32, -1, 4, "pernode"),
    ("rng_reference", 1024, 32, 0, 2, "reference"),
])
def test_invalid_shard_options(gpu, clean, what, n, min_size, rank, count, rng_mode):
    """Rejected with BGP_ERR_INVALID, no shard ranges reported, and the handle computes the next problem as a fresh
    one does."""
    lib = _lib().load()
    kernel, x, yerr, _ = _problem("exp", n)
    s = _native()
    # first a valid sharded compute, so that stale ranges would show
    _lib().check(_compute_status(s, kernel, x, yerr, min_size=32, tol=1e-12, shard_rank=0, shard_count=2))
    st = _compute_status(s, kernel, x, yerr, min_size=min_size, tol=1e-12, rng_mode=rng_mode, shard_rank=rank,
                         shard_count=count)
    assert st == BGP_ERR_INVALID, what
    assert not lib.bgp_hodlr_computed(s._ptr)
    row0, rows = C.c_int64(), C.c_int64()
    assert lib.bgp_hodlr_shard_rows(s._ptr, 0, C.byref(row0), C.byref(rows)) == BGP_ERR_INDEX
    _lib().check(_compute_status(s, kernel, x, yerr, min_size=32, tol=1e-12))
    fresh = _single(kernel, x, yerr, min_size=32, tol=1e-12)
    assert s.nodes() == fresh.nodes()
    assert abs(s.log_determinant - fresh.log_determinant) <= REUSE_TOL * max(1.0, abs(fresh.log_determinant))


def test_a_compute_rejected_on_its_inputs_ends_the_exchange(gpu, clean):
    """bgp_hodlr_compute rejects an input with no dimensions before it factors anything.  After a host-exchange
    compute that must still drop the shard ranges and the pending top step: otherwise finish_top would mark the handle
    computed with the previous problem's factorisation."""
    lib = _lib().load()
    kernel, x, yerr, _ = _problem("exp", 1024)
    s = _native()
    _lib().check(_compute_status(s, kernel, x, yerr, min_size=32, tol=1e-12, shard_rank=0, shard_count=2))
    assert _shard_rows(s, 2) == [(0, 512), (512, 512)]
    assert _compute_status(s, kernel, np.zeros((1024, 0)), yerr, min_size=32, tol=1e-12, shard_rank=0,
                           shard_count=2) == BGP_ERR_INVALID
    row0, rows = C.c_int64(), C.c_int64()
    assert lib.bgp_hodlr_shard_rows(s._ptr, 0, C.byref(row0), C.byref(rows)) == BGP_ERR_INDEX
    buf = _Dev(2 * 512 * 512)
    assert lib.bgp_hodlr_export_top(s._ptr, buf.p, 512) == BGP_ERR_NOT_COMPUTED
    assert lib.bgp_hodlr_import_top(s._ptr, buf.p, 512) == BGP_ERR_NOT_COMPUTED
    assert lib.bgp_hodlr_finish_top(s._ptr) == BGP_ERR_NOT_COMPUTED
    assert not lib.bgp_hodlr_computed(s._ptr)
