# -*- coding: utf-8 -*-
"""
``HODLRSolver`` — the O(N log^2 N) solver plugin, on the H100.

Drop-in for the reference's shim ``src/george/solvers/hodlr.py:12-76``: same constructor defaults
(``min_size=100, tol=0.1, seed=42``), ``compute`` builds a fresh native solver, ``apply_sqrt`` raises
``NotImplementedError``, pickling drops the native handle and clears ``computed`` so the GP refactorises lazily.
"""

import numpy as np

from .basic import BasicSolver
from ._hodlr import HODLRSolver as HODLRSolverInterface

__all__ = ["HODLRSolver"]

FISHER_HODLR = ("the Fisher information is not implemented for the HODLR solvers: its exact trace is O(P N^3) at HODLR "
                "sizes; use the dense BasicSolver")


class HODLRSolver(BasicSolver):

    # no batched HODLR factorisation: GP.batch_log_likelihood, GP.batch_predict, GP.batch_grad_log_likelihood,
    # GP.batch_sample_conditional, GP.batch_grad_predict and the GP.batch_*loo* methods take their per-vector loops;
    # GP.batch_fisher_information raises NotImplementedError, as GP.fisher_information does
    batch_log_likelihood = None
    batch_predict = None
    batch_grad_terms = None
    batch_sample = None
    batch_predict_grad = None
    batch_loo_terms = None
    batch_fisher_terms = None

    def __init__(self, kernel, min_size=100, tol=0.1, seed=42, rng_mode=None, rank_capacity=0,
                 exhaust="dense"):
        # rng_mode=None: the reference's single shared mt19937 (bit-for-bit its pivot order) whenever the tolerance is
        # loose enough for the answer to DEPEND on the pivots (tol > 1e-6; the reference's default is 0.1), the
        # level-parallel per-node streams otherwise (the answer then agrees with the reference's far inside 1e-6)
        self.min_size = min_size
        self.tol = tol
        self.seed = seed
        self.rng_mode = rng_mode
        self.rank_capacity = rank_capacity
        self.exhaust = exhaust
        super(HODLRSolver, self).__init__(kernel)

    def compute(self, x, yerr):
        self.solver = HODLRSolverInterface()
        self.solver.compute(self.kernel, x, yerr, self.min_size, self.tol, self.seed, rng_mode=self.rng_mode,
                            rank_capacity=self.rank_capacity, exhaust=self.exhaust)
        self._log_det = self.solver.log_determinant
        self.computed = self.solver.computed

    def apply_inverse(self, y, in_place=False):
        return self.solver.apply_inverse(y, in_place=in_place)

    def dot_solve(self, y):
        return self.solver.dot_solve(y)

    def apply_sqrt(self, r):
        raise NotImplementedError("apply_sqrt is not implemented for the HODLRSolver")

    def get_inverse(self):
        return self.solver.get_inverse()

    def _require(self):
        if getattr(self, "solver", None) is None or not self._computed:
            raise RuntimeError("you must call 'compute' first")
        self._n, self._ndim = self.solver._n, self.solver._ndim

    def _grad_terms_call(self, which, r, alpha, g, diag):
        return self.solver._lib.bgp_hodlr_grad_terms(self.solver._ptr, which, r, alpha, g, diag)

    def _grad_x_terms_lib(self, *args):
        return self.solver._lib.bgp_hodlr_grad_x_terms(self.solver._ptr, *args)

    def fisher_terms(self, r, which, v, prod_ms=None):
        """The Fisher information is not available on a HODLR factorisation: its exact trace needs N^2 products, O(P N^3)
        at HODLR sizes.  Raises ``NotImplementedError`` (``GP.fisher_information`` raises it before any device work)."""
        raise NotImplementedError(FISHER_HODLR)

    def _loo_terms_call(self, which, r, alpha, d, beta, g, diag):
        return self.solver._lib.bgp_hodlr_loo_terms(self.solver._ptr, which, r, alpha, d, beta, g, diag)

    def predictive(self, kernel, xs, what):
        """``BasicSolver.predictive`` on the HODLR factorisation (``include/bgp.h: bgp_hodlr_predict``); ``None`` on a
        sharded factorisation."""
        self._require()
        if self.solver.shard_count > 1:
            return None
        return self._predictive_call(self.solver._lib.bgp_hodlr_predict, self.solver._ptr, kernel, xs, what)

    def predictive_grad(self, kernel, xs):
        """``BasicSolver.predictive_grad`` on the HODLR factorisation (``include/bgp.h: bgp_hodlr_predict_grad``);
        ``None`` on a sharded factorisation."""
        self._require()
        if self.solver.shard_count > 1:
            return None
        return self._predictive_grad_call(self.solver._lib.bgp_hodlr_predict_grad, self.solver._ptr, kernel, xs)

    def sample_predictive(self, kernel, xs, mean, z, jitter):
        """``BasicSolver.sample_predictive`` on the HODLR factorisation (``include/bgp.h: bgp_hodlr_sample``); ``None``
        on a sharded factorisation."""
        self._require()
        if self.solver.shard_count > 1:
            return None
        return self._sample_call(self.solver._lib.bgp_hodlr_sample, self.solver._ptr, kernel, xs, mean, z, jitter)

    def sample_prior(self, z):
        """Prior draws at the computed coordinates without the mean: ``(W z^T)^T`` for ``z`` of shape ``(size, N)``,
        ``W`` the symmetric factor ``K~ = W W^T`` of the HODLR matrix (``HODLRSolverInterface.apply_symmetric_factor``);
        ``None`` on a sharded factorisation."""
        self._require()
        if self.solver.shard_count > 1:
            return None
        z = np.asarray(z, dtype=np.float64)
        if z.shape[0] == 0:
            return np.empty(z.shape, dtype=np.float64)
        return np.ascontiguousarray(self.solver.apply_symmetric_factor(z.T).T)

    def __getstate__(self):
        state = self.__dict__.copy()
        state["_computed"] = False
        state["_handle"] = None
        state.pop("solver", None)
        return state

    def __setstate__(self, state):
        self.__dict__.update(state)
