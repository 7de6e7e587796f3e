# -*- coding: utf-8 -*-
"""
Multi-GPU HODLR: one process per GPU, the tree sharded by top-level sub-tree (SURVEY.md §8e).

The reference has no distributed code; what shards is the algorithmic independence of HODLR sub-trees
(``hodlr.h:58-61,78-79``): below depth ``log2(P)`` the ``P`` sub-trees of ``~N/P`` points never touch each other's rows
(``hodlr.h:95-102,240-253``).  Each rank

1. factors its own sub-tree (leaves, ACAs, up-sweep) and applies it to ITS rows of the ``log2(P)`` top-level factor
   panels (whose ACAs every rank recomputes redundantly from the replicated coordinates — no communication);
2. takes part in ONE all-gather of those locally-solved row slices — the only data-path collective of ``compute`` —
   issued by the library itself on the solver's stream (``csrc/comm.cu``: pack kernel -> ``ncclAllGather`` -> unpack
   kernels, no host round trip);
3. finishes the ``P - 1`` top nodes redundantly (Gram, 2r x 2r LU, log-det, update).

``log|K|`` is an all-reduce of one double; a solve is: local sub-tree solve on the owned slice, one all-gather of the
vector, top nodes redundantly.  The log-likelihood gradient (``grad_terms``) is that solve for alpha, each rank
streaming K^-1 over the columns of its own rows, an all-reduce of ``g`` and an all-gather of the diagonal.  The
predictive variance / covariance (``predictive``) solves K(x, x*) chunk by chunk, each rank building its own rows and
contracting over them, and ends with one all-reduce of the result.
``torch.distributed`` is plumbing only: it broadcasts the 128-byte NCCL unique id with
which every rank initialises the library's communicator (``ensure_device_comm``).  All arithmetic and all data-path
collectives are in ``csrc/hodlr.cu`` / ``csrc/comm.cu``.

The exchange helpers at the bottom are backend-agnostic (tested with gloo on CPU tensors in ``tests/test_parallel.py``).
"""

import ctypes as C

import numpy as np

from . import _lib
from ._spec import flatten
from .solvers.basic import BasicSolver, _grad_x_terms_call
from .solvers.hodlr import FISHER_HODLR

__all__ = ["ShardedHODLRSolver", "shard_ranges", "allgather_padded"]


def shard_ranges(n, shard_count, min_size):
    """Row ranges ``[(start, size), ...]`` of the depth-``log2(shard_count)`` nodes of the reference tree
    (``hodlr.h:48-61``: ``half = size // 2``; a node splits iff ``half >= min_size``), or ``None`` when the tree is
    too shallow to be cut that many ways."""
    if shard_count < 1 or shard_count & (shard_count - 1):
        raise ValueError("shard_count must be a power of two")
    level = [(0, int(n))]
    cut = shard_count.bit_length() - 1
    for _ in range(cut):
        nxt = []
        for start, size in level:
            half = size // 2
            if half < min_size:
                return None
            nxt.append((start, half))
            nxt.append((start + half, size - half))
        level = nxt
    return level


def allgather_padded(local, rows_pad, group=None):
    """All-gather 2-D blocks ``local`` (cols x rows_i, last dim contiguous) whose row counts differ by at most a few:
    every rank pads to ``rows_pad`` and the result has shape ``(world, cols, rows_pad)``."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group)
    cols, rows = local.shape
    send = local
    if rows != rows_pad:
        send = torch.zeros((cols, rows_pad), dtype=local.dtype, device=local.device)
        send[:, :rows] = local
    send = send.contiguous()
    out = torch.empty((world, cols, rows_pad), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out.view(-1), send.view(-1), group=group)
    return out


_COMM_WORLD = 0


def ensure_device_comm(group=None):
    """Create (once) the NCCL communicator libbgp_b200 issues its data-path collectives on (``csrc/comm.cu``): rank 0
    makes the unique id, it is broadcast over the host's process group, every rank initialises.  Returns the world size."""
    global _COMM_WORLD
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group)
    if world == 1 or _COMM_WORLD == world:
        return world
    lib = _lib.load()
    rank = dist.get_rank(group)
    buf = (C.c_ubyte * 128)()
    path = None
    try:
        import nvidia.nccl
        import glob
        import os
        hits = glob.glob(os.path.join(os.path.dirname(nvidia.nccl.__file__), "lib", "libnccl.so*"))
        path = hits[0].encode() if hits else None
    except Exception:
        path = None
    if rank == 0:
        _lib.check(lib.bgp_comm_unique_id(buf, path))
    dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend(group) == "nccl" else torch.device("cpu")
    t = torch.tensor(list(bytes(buf)), dtype=torch.uint8, device=dev)
    dist.broadcast(t, src=0, group=group)
    ident = (C.c_ubyte * 128)(*t.cpu().tolist())
    _lib.check(lib.bgp_comm_init(ident, rank, world, path))
    _COMM_WORLD = world
    return world


class ShardedHODLRSolver(object):
    """Solver plugin with the ``HODLRSolver`` surface whose ``compute``/``dot_solve`` are collective over a
    ``torch.distributed`` process group (one rank per GPU).  ``x``, ``yerr`` and ``y`` are replicated on every rank."""

    def __init__(self, kernel, min_size=100, tol=0.1, seed=42, rank_capacity=0, exhaust="dense", group=None):
        self.kernel = kernel
        self.min_size, self.tol, self.seed = min_size, tol, seed
        self.rank_capacity, self.exhaust, self.group = rank_capacity, exhaust, group
        self._computed = False
        self._log_det = None
        self.solver = None

    @property
    def computed(self):
        return self._computed

    @property
    def log_determinant(self):
        return self._log_det

    def compute(self, x, yerr):
        import torch.distributed as dist
        from .solvers._hodlr import HODLRSolver as Native
        rank, world = dist.get_rank(self.group), dist.get_world_size(self.group)
        x = np.ascontiguousarray(x, dtype=np.float64)
        if x.ndim == 1:
            x = x[:, None]
        yerr = np.ascontiguousarray(yerr, dtype=np.float64)
        self._n = x.shape[0]
        self._ranges = shard_ranges(self._n, world, self.min_size)
        if self._ranges is None:
            raise ValueError("the HODLR tree (N={0}, min_size={1}) is too shallow to shard {2} ways".format(
                self._n, self.min_size, world))
        if ensure_device_comm(self.group) != world:
            raise RuntimeError("the library's NCCL communicator does not span the process group")
        if self.solver is None:
            self.solver = Native()  # one handle for the life of the solver: buffers and rank capacities are reused
        # collective: local sub-tree, all-gather of the top panel rows, top nodes, log-det all-reduce (csrc/hodlr.cu)
        self.solver.compute(self.kernel, x, yerr, self.min_size, self.tol, self.seed, rank_capacity=self.rank_capacity,
                            shard_rank=rank, shard_count=world, exhaust=self.exhaust)
        self._log_det = self.solver.log_determinant
        self._computed = True

    def apply_inverse(self, y, in_place=False):
        """Collective; ``y`` replicated on every rank."""
        return self.solver.apply_inverse(y, in_place=in_place)

    def dot_solve(self, y):
        """Collective; ``y`` replicated on every rank."""
        return self.solver.dot_solve(y)

    def grad_terms(self, r, which):
        """``(alpha, g, diagA)`` for ``GP.grad_log_likelihood``, as ``BasicSolver.grad_terms`` returns them.
        Collective; ``r`` replicated on every rank.  Each rank streams K^-1 over the columns of its own rows; the only
        collectives are the solve for alpha, an all-reduce of ``g`` and an all-gather of the diagonal
        (``include/bgp.h: bgp_hodlr_grad_terms``).  K^-1 is never formed."""
        if self.solver is None or not self._computed:
            raise RuntimeError("you must call 'compute' first")
        r = np.ascontiguousarray(r, dtype=np.float64)
        if r.shape != (self._n,):
            raise ValueError("dimension mismatch")
        which = np.ascontiguousarray(which, dtype=np.uint32)
        alpha = np.empty(self._n, dtype=np.float64)
        g = np.zeros(max(which.size, 1), dtype=np.float64)
        diag = np.empty(self._n, dtype=np.float64)
        lib = self.solver._lib
        _lib.check(lib.bgp_hodlr_grad_terms(self.solver._ptr, _lib.ptr(which), _lib.ptr(r), _lib.ptr(alpha),
                                            _lib.ptr(g), _lib.ptr(diag)))
        return alpha, g[:which.size], diag

    def grad_x_terms(self, r, which):
        """``(alpha, g, diagA, dx)`` for ``GP.grad_log_likelihood_x``, as ``BasicSolver.grad_x_terms`` returns them.
        Collective; ``r`` replicated on every rank, and every rank returns the same result.  Each rank streams K^-1 over
        the columns of its own rows and contracts their input gradient in the same pass; the collectives are those of
        :func:`grad_terms` and one all-gather of the ``dx`` row slices (``include/bgp.h: bgp_hodlr_grad_x_terms``).
        The argument checks run on every rank before any collective, so a bad call leaves no rank waiting."""
        if self.solver is None or not self._computed:
            raise RuntimeError("you must call 'compute' first")
        lib, ptr = self.solver._lib, self.solver._ptr
        return _grad_x_terms_call(lambda *args: lib.bgp_hodlr_grad_x_terms(ptr, *args), self._n, self.solver._ndim,
                                  r, which)

    def loo_terms(self, r, which=None):
        """Leave-one-out cross-validation is not available on a sharded factorisation: its gradient would need a
        collective full solve per slab.  Raises ``NotImplementedError`` on every rank before any collective, so no rank
        is left waiting."""
        raise NotImplementedError("leave-one-out cross-validation is not implemented for the ShardedHODLRSolver")

    def fisher_terms(self, r, which, v, prod_ms=None):
        """The Fisher information is not available on a sharded factorisation, as on ``HODLRSolver``.  Raises
        ``NotImplementedError`` on every rank before any collective, so no rank is left waiting."""
        raise NotImplementedError(FISHER_HODLR)

    def predictive(self, kernel, xs, what):
        """``BasicSolver.predictive`` on the sharded factorisation: the variance (``what="var"``, ``(ns,)``) or
        covariance (``"cov"``, ``(ns, ns)``) of ``GP.predict``.  Collective; ``xs`` replicated on every rank, and every
        rank returns the same result.  Each rank builds and contracts K(x, x*) over its own rows only; the collectives
        are the chunks' solves and one all-reduce of the result (``include/bgp.h: bgp_hodlr_predict``)."""
        if self.solver is None or not self._computed:
            raise RuntimeError("you must call 'compute' first")
        return BasicSolver._predictive_call(self.solver._lib.bgp_hodlr_predict, self.solver._ptr, kernel, xs, what)

    def predictive_grad(self, kernel, xs):
        """``BasicSolver.predictive_grad`` on the sharded factorisation: ``(var, dvar)`` for ``GP.grad_predict``, ``var``
        bit for bit what :func:`predictive` returns for ``"var"``.  Collective; ``xs`` replicated on every rank, and every
        rank returns the same result.  Each rank builds and contracts K(x, x*) and its test-point gradient over its own
        rows only; the collectives are the chunks' solves and two all-reduces, ``var``'s as in :func:`predictive` and then
        ``dvar``'s (``include/bgp.h: bgp_hodlr_predict_grad``)."""
        if self.solver is None or not self._computed:
            raise RuntimeError("you must call 'compute' first")
        return BasicSolver._predictive_grad_call(self.solver._lib.bgp_hodlr_predict_grad, self.solver._ptr, kernel, xs)

    def apply_symmetric_factor(self, z, transpose=False):
        """``W z`` (or ``W^T z`` with ``transpose``) for the symmetric factor ``K~ = W W^T`` of the sharded
        factorisation, as ``HODLRSolver.apply_symmetric_factor``: ``z`` of shape ``(N,)`` or ``(N, k)``, the result of
        the same shape.  Collective; ``z`` replicated on every rank, and every rank returns the same result.  The factor
        is built on the first call after a ``compute``: each rank its own sub-tree's rows, one all-gather of those rows
        of the top levels' columns, the top nodes on every rank; an apply is the top levels, the rank's own levels and
        leaves, and one all-gather per 64 columns (``include/bgp.h: bgp_hodlr_sym_apply``).  A ``K~`` that is not
        positive definite raises ``numpy.linalg.LinAlgError`` on every rank."""
        if self.solver is None or not self._computed:
            raise RuntimeError("you must call 'compute' first")
        z = np.asarray(z, dtype=np.float64)
        if z.ndim not in (1, 2) or z.shape[0] != self._n:
            raise ValueError("dimension mismatch")
        b = np.array(z.reshape(self._n, -1), dtype=np.float64, order="F")
        _lib.check(self.solver._lib.bgp_hodlr_sym_apply(self.solver._ptr, _lib.ptr(b), b.shape[1], self._n,
                                                        1 if transpose else 0))
        return b.reshape(z.shape)

    @property
    def symmetric_log_determinant(self):
        """``log|K~|`` from the symmetric factor, the same on every rank (one all-reduce of the ranks' partial sums).
        Collective (``include/bgp.h: bgp_hodlr_sym_log_determinant``)."""
        if self.solver is None or not self._computed:
            raise RuntimeError("you must call 'compute' first")
        out = C.c_double()
        _lib.check(self.solver._lib.bgp_hodlr_sym_log_determinant(self.solver._ptr, C.byref(out)))
        return out.value

    def apply_sqrt(self, r):
        raise NotImplementedError("apply_sqrt is not implemented for the HODLRSolver")

    def get_inverse(self):
        return self.solver.get_inverse()
