# -*- coding: utf-8 -*-
"""
``_hodlr.HODLRSolver`` — the native HODLR interface, same surface as the reference's pybind11 class
(``src/george/solvers/_hodlr.cpp:115-204``): ``compute(kernel_spec, x, yerr, min_size=100, tol=0.1, seed=42)``,
``apply_inverse(x, in_place=False)`` (returns ``(n, 1)`` for a vector, like the Eigen caster does),
``dot_solve(x)``, ``get_inverse()``, read-only ``computed`` and ``log_determinant``.

Everything numeric happens in ``csrc/hodlr.cu`` on the H100.  Extra keyword-only knobs (not in the reference):
``rng_mode`` ("pernode" | "reference"), ``rank_capacity``, ``exhaust`` ("dense" | "lowrank", see
``include/bgp.h: bgp_hodlr_opts_t.exhaust_mode``).
"""

import ctypes as C

import numpy as np

from .. import _lib
from .._spec import HodlrNodeInfo, HodlrOpts, flatten

RNG_MODES = {"pernode": 0, "reference": 1}


def resolve_rng_mode(rng_mode, tol):
    """``None`` -> the reference's own stream order when the result depends on the pivots (``tol > 1e-6``; at the
    reference's default ``tol = 0.1`` the HODLR answer is 3e-3 away from the dense one, SURVEY.md App. A), the
    level-parallel per-node streams when it does not."""
    if rng_mode is None:
        return "reference" if tol > 1e-6 else "pernode"
    return rng_mode
EXHAUST_MODES = {"dense": 0, "lowrank": 1}


class HODLRSolver(object):

    # Native handles outlive the Python objects that use them.  The reference builds a brand-new solver on every
    # ``GP.compute`` (gp.py:327); a native handle is only device buffers, the rank capacities its last factorisation
    # ended with and the instantiated CUDA graph of the ACA loop, all of which the next compute() of the same shape
    # reuses — so a dying solver parks its handle here and the next one picks it up (state is overwritten by compute()).
    _parked = []
    _max_parked = 2

    def __init__(self):
        self._lib = _lib.load()
        if HODLRSolver._parked:
            self._ptr = HODLRSolver._parked.pop()
        else:
            self._ptr = C.c_void_p()
            _lib.check(self._lib.bgp_hodlr_create(C.byref(self._ptr)))
        self._n = 0
        self.shard_count = 1
        self._fresh = True  # nothing computed through THIS object yet (a parked handle still holds its previous state)

    def __del__(self):
        if getattr(self, "_ptr", None) is not None and self._ptr:
            try:
                if len(HODLRSolver._parked) < HODLRSolver._max_parked:
                    HODLRSolver._parked.append(self._ptr)
                else:
                    self._lib.bgp_hodlr_destroy(self._ptr)
            except Exception:  # interpreter shutdown
                pass
            self._ptr = None

    @classmethod
    def release_parked(cls):
        """Destroy the parked native handles (frees their device buffers)."""
        lib = _lib.load()
        while cls._parked:
            lib.bgp_hodlr_destroy(cls._parked.pop())

    @property
    def computed(self):
        if self._fresh:
            return 0
        return int(self._lib.bgp_hodlr_computed(self._ptr))

    @property
    def log_determinant(self):
        if self._fresh:
            raise RuntimeError("the solver has not been computed")
        out = C.c_double()
        _lib.check(self._lib.bgp_hodlr_log_determinant(self._ptr, C.byref(out)))
        return out.value

    def _opts(self, min_size, tol, seed, rng_mode, rank_capacity, shard_rank=0, shard_count=1, exhaust="dense"):
        o = HodlrOpts()
        self._lib.bgp_hodlr_default_opts(C.byref(o))
        o.min_size, o.tol, o.seed = int(min_size), float(tol), int(seed)
        o.rng_mode = RNG_MODES[rng_mode] if isinstance(rng_mode, str) else int(rng_mode)
        o.rank_capacity = int(rank_capacity)
        o.shard_rank, o.shard_count = int(shard_rank), int(shard_count)
        o.exhaust_mode = EXHAUST_MODES[exhaust] if isinstance(exhaust, str) else int(exhaust)
        return o

    def compute(self, kernel_spec, x, yerr, min_size=100, tol=0.1, seed=42, rng_mode=None, rank_capacity=0,
                shard_rank=0, shard_count=1, exhaust="dense"):
        rng_mode = "pernode" if shard_count > 1 and rng_mode is None else resolve_rng_mode(rng_mode, tol)
        x = np.ascontiguousarray(x, dtype=np.float64)
        if x.ndim != 2:
            raise ValueError("array has incorrect number of dimensions: {0}; expected 2".format(x.ndim))
        yerr = np.ascontiguousarray(yerr, dtype=np.float64)
        if yerr.shape != (x.shape[0],):
            raise ValueError("dimension mismatch")
        spec = flatten(kernel_spec)
        o = self._opts(min_size, tol, seed, rng_mode, rank_capacity, shard_rank, shard_count, exhaust)
        self._n = x.shape[0]
        self.shard_count = int(shard_count)
        self._fresh = False
        _lib.check(self._lib.bgp_hodlr_compute(self._ptr, C.byref(spec), _lib.ptr(x), x.shape[0], x.shape[1],
                                               _lib.ptr(yerr), C.byref(o)))
        return 0

    def _require_computed(self):
        if self._fresh:
            raise RuntimeError("the solver has not been computed")

    def apply_inverse(self, x, in_place=False):
        self._require_computed()
        x = np.asarray(x)
        if in_place and x.dtype == np.float64 and x.flags.f_contiguous and x.flags.writeable and x.ndim == 2:
            b = x
        else:
            b = np.array(x, dtype=np.float64, order="F")
            if b.ndim == 1:
                b = b.reshape(-1, 1, order="F")
        if b.shape[0] != self._n:
            raise ValueError("dimension mismatch")
        _lib.check(self._lib.bgp_hodlr_apply_inverse(self._ptr, _lib.ptr(b), b.shape[1], self._n))
        if in_place and b is not x:
            x[...] = b.reshape(x.shape)
        return b

    def dot_solve(self, x):
        self._require_computed()
        x = np.ascontiguousarray(x, dtype=np.float64)
        if x.shape != (self._n,):
            raise ValueError("dimension mismatch")
        out = C.c_double()
        _lib.check(self._lib.bgp_hodlr_dot_solve(self._ptr, _lib.ptr(x), C.byref(out)))
        return out.value

    def get_inverse(self):
        self._require_computed()
        # the library solves against a COLUMN-major identity; the HODLR inverse is symmetric only to `tol`, so hand the
        # buffer back with the orientation the reference's Eigen -> numpy conversion has (_hodlr.cpp:193-199): M[i, j]
        out = np.empty((self._n, self._n), dtype=np.float64)
        _lib.check(self._lib.bgp_hodlr_get_inverse(self._ptr, _lib.ptr(out)))
        return out.T

    # ---- introspection (tree / index structure; not in the reference) -------------------------------------------
    def nodes(self):
        n = C.c_int64()
        _lib.check(self._lib.bgp_hodlr_num_nodes(self._ptr, C.byref(n)))
        arr = (HodlrNodeInfo * n.value)()
        _lib.check(self._lib.bgp_hodlr_node_info(self._ptr, arr))
        names = [f[0] for f in HodlrNodeInfo._fields_]
        return [dict((k, getattr(a, k)) for k in names) for a in arr]

    def pivots(self, node, rank):
        rows = np.zeros(max(rank, 1), dtype=np.int32)
        cols = np.zeros(max(rank, 1), dtype=np.int32)
        _lib.check(self._lib.bgp_hodlr_node_pivots(self._ptr, node, _lib.ptr(rows), _lib.ptr(cols)))
        return rows[:rank], cols[:rank]

    def factors(self, node):
        """``(Vl, Ur)``: the ACA factors of internal node ``node`` (pre-order index), ``(half, rank)`` and
        ``(size - half, rank)``, with ``K[right, left] ~ Ur @ Vl.T`` (``include/bgp.h: bgp_hodlr_node_factors``)."""
        self._require_computed()
        nodes = self.nodes()
        if not 0 <= node < len(nodes):
            raise IndexError("node index out of range")
        nd = nodes[node]
        out = np.zeros((nd["size"], nd["rank"]), dtype=np.float64, order="F")
        _lib.check(self._lib.bgp_hodlr_node_factors(self._ptr, node, _lib.ptr(out)))
        return out[:nd["half"]], out[nd["half"]:]

    def draw_paths(self):
        """How often the last compute's speculative row draws left the common path
        (``include/bgp.h: bgp_hodlr_last_draw_paths``)."""
        self._require_computed()
        c = (C.c_uint64 * 4)()
        _lib.check(self._lib.bgp_hodlr_last_draw_paths(self._ptr, c))
        return dict(zip(("lemire_redos", "truncated_batches", "sequential_draws", "partial_commits"), (int(v) for v in c)))

    def eval_units(self):
        """The last compute's candidate-evaluation work units: ``pulled`` by the evaluation kernel and ``live`` (at
        least one candidate evaluated) (``include/bgp.h: bgp_hodlr_last_eval_units``)."""
        self._require_computed()
        c = (C.c_uint64 * 2)()
        _lib.check(self._lib.bgp_hodlr_last_eval_units(self._ptr, c))
        return dict(zip(("pulled", "live"), (int(v) for v in c)))

    def timing(self):
        t = (C.c_double * 5)()
        _lib.check(self._lib.bgp_hodlr_last_timing(self._ptr, t))
        return dict(zip(("leaves_ms", "aca_ms", "upsweep_ms", "compute_ms", "solve_ms"), list(t)))

    def grad_timing(self):
        """The last ``grad_terms`` call (``include/bgp.h: bgp_hodlr_last_grad_timing``): ``solve_ms`` and
        ``contract_ms`` (measured with profiling on, 0 otherwise), ``slabs`` and ``slab_cols`` (0 on the resident
        path)."""
        t = (C.c_double * 4)()
        _lib.check(self._lib.bgp_hodlr_last_grad_timing(self._ptr, t))
        out = dict(zip(("solve_ms", "contract_ms", "slabs", "slab_cols"), list(t)))
        out["slabs"], out["slab_cols"] = int(out["slabs"]), int(out["slab_cols"])
        return out

    def grad_terms_local(self, alpha_dev, which, diag_dev=None):
        """This handle's part of the streamed gradient (``include/bgp.h: bgp_hodlr_grad_terms_local_dev``): the partial
        ``g`` (``(len(which),)``) over the columns of its own rows, from ``alpha_dev``, a device pointer to the full
        ``K^-1 r``.  ``diag_dev`` (a device pointer to ``n`` doubles, or ``None``) receives ``alpha_j^2 - K^-1_jj`` for
        those rows only.  Issues no collective."""
        self._require_computed()
        which = np.ascontiguousarray(which, dtype=np.uint32)
        g = np.zeros(max(which.size, 1), dtype=np.float64)
        _lib.check(self._lib.bgp_hodlr_grad_terms_local_dev(self._ptr, _lib.ptr(which), alpha_dev, _lib.ptr(g),
                                                            diag_dev))
        return g[:which.size]

    def set_profiling(self, on=True):
        _lib.check(self._lib.bgp_hodlr_set_profiling(self._ptr, 1 if on else 0))

    def aca_profile(self):
        p = (C.c_double * 12)()
        _lib.check(self._lib.bgp_hodlr_last_aca_profile(self._ptr, p))
        out = dict(zip(("eval_ms", "eval_launches", "evals", "update_fmas", "candidates", "evaluated"), list(p)[:6]))
        out["kernel_ms"] = dict(zip(("a2_eval", "a2_decide", "a2_vrow", "a2_pivot", "a2_vnorm_ucol", "a2_finish"), list(p)[6:]))
        return out

    def work(self):
        w = (C.c_double * 6)()
        _lib.check(self._lib.bgp_hodlr_last_work(self._ptr, w))
        return dict(zip(("evals", "bytes", "flops", "R", "leaf", "levels"), list(w)))
