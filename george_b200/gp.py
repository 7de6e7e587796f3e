# -*- coding: utf-8 -*-
"""
The ``GP`` object: caller of the accelerated path.

Behavioural mirror of the reference's ``src/george/gp.py:22-643`` (same constructor, methods, caching and error
semantics) — ``compute`` hands ``(x, sqrt(yerr^2 + exp(white_noise)))`` to a freshly built solver plugin
(``gp.py:303-337``), ``log_likelihood`` is ``_const - 0.5 * solver.dot_solve(y - mean)`` (``gp.py:369-397``) and
``predict`` reuses the factorisation (``gp.py:482-545``).  All O(N^2)/O(N log^2 N) work happens inside the solver
plugins on the H100; this file is host bookkeeping.
"""

import ctypes as C
import warnings

import numpy as np
from numpy.linalg import LinAlgError

from . import _lib, kernels
from ._spec import flatten, num_params, patch_specs
from .modeling import ConstantModel, ModelSet
from .solvers import BasicSolver, TrivialSolver
from .solvers.basic import NONFINITE_RHS
from .utils import multivariate_gaussian_samples

__all__ = ["GP"]

# jitter added to the diagonal when no observational uncertainty is given (reference gp.py:19)
TINY = 1.25e-12
# most kernel parameters the device gradient contraction takes (include/bgp.h)
_MAX_GRAD_PARAMS = 64


def _as_model(obj):
    """Scalars become ConstantModel; anything else is assumed to follow the modeling protocol."""
    try:
        value = float(obj)
    except TypeError:
        return obj
    return ConstantModel(float(value))


def _is_number(obj):
    try:
        float(obj)
    except TypeError:
        return False
    return True


class GP(ModelSet):
    """Gaussian-process regression model.

    :param kernel: a :class:`kernels.Kernel` (default: ``EmptyKernel``)
    :param fit_kernel: include the kernel parameters in the parameter vector (default ``True``)
    :param mean: scalar, callable-model or modeling-protocol object (default ``0``)
    :param fit_mean: fit the mean parameters (default: only when a non-scalar mean is given)
    :param white_noise: log of the white-noise variance added on the diagonal (default ``log(TINY)``)
    :param fit_white_noise: fit the white-noise parameters
    :param solver: solver plugin class (default ``BasicSolver``, or ``TrivialSolver`` without a kernel)
    :param kwargs: forwarded to the solver constructor (e.g. ``min_size``, ``tol``, ``seed`` for ``HODLRSolver``)
    """

    def __init__(self, kernel=None, fit_kernel=True, mean=None, fit_mean=None, white_noise=None,
                 fit_white_noise=None, solver=None, **kwargs):
        self._computed = False
        self._alpha = None
        self._y = None

        super(GP, self).__init__([
            ("mean", ConstantModel(0.0) if mean is None else _as_model(mean)),
            ("white_noise", ConstantModel(np.log(TINY)) if white_noise is None else _as_model(white_noise)),
            ("kernel", kernels.EmptyKernel() if kernel is None else kernel),
        ])

        # a plain number for mean / white_noise is not fitted unless asked for
        if _is_number(mean) and fit_mean is None:
            fit_mean = False
        if _is_number(white_noise) and fit_white_noise is None:
            fit_white_noise = False

        if not fit_kernel:
            self.models["kernel"].freeze_all_parameters()
        if mean is None or (fit_mean is not None and not fit_mean):
            self.models["mean"].freeze_all_parameters()
        if white_noise is None or (fit_white_noise is not None and not fit_white_noise):
            self.models["white_noise"].freeze_all_parameters()

        if solver is None:
            no_kernel = kernel is None or kernel.kernel_type == kernels.EmptyKernel.kernel_type
            solver = TrivialSolver if no_kernel else BasicSolver
        self.solver_type = solver
        self.solver_kwargs = kwargs
        self.solver = None

    # -- sub-models ------------------------------------------------------------------------------------------------
    @property
    def mean(self):
        return self.models["mean"]

    @property
    def white_noise(self):
        return self.models["white_noise"]

    @staticmethod
    def _model_input(x):
        return x[:, 0] if (x.ndim == 2 and x.shape[1] == 1) else x

    def _call_mean(self, x):
        mu = self.mean.get_value(self._model_input(x)).flatten()
        if not np.all(np.isfinite(mu)):
            raise ValueError("mean function returned NaN or Inf for parameters:\n{0}".format(
                self.mean.get_parameter_dict(include_frozen=True)))
        return mu

    def _call_mean_gradient(self, x):
        g = self.mean.get_gradient(self._model_input(x))
        if np.any(np.isnan(g)) or np.any(np.isinf(g)):
            raise ValueError("mean gradient function returned NaN or Inf for parameters:\n{0}".format(
                self.mean.get_parameter_dict(include_frozen=True)))
        return g

    def _call_white_noise(self, x):
        return self.white_noise.get_value(self._model_input(x)).flatten()

    # Constant mean / white-noise models (the defaults) need no per-point array: at N ~ 10^5..10^6 every extra pass
    # over an N-vector on the host costs about as much as a level of the factorisation on the device.
    def _constant_of(self, model):
        return float(model.value) if type(model) is ConstantModel else None

    def _sigma(self, x):
        """sqrt(yerr^2 + exp(white_noise(x)))  (reference gp.py:330)."""
        c = self._constant_of(self.white_noise)
        if c is None:
            return np.sqrt(self._yerr2 + np.exp(self._call_white_noise(x)))
        sigma = self._yerr2 + np.exp(c)
        return np.sqrt(sigma, out=sigma)

    def _residual_of(self, y):
        """y - mean(x) as a contiguous float64 vector (reference gp.py:388-393); raises on a non-finite mean."""
        c = self._constant_of(self.mean)
        if c is None:
            return np.ascontiguousarray(self._check_dimensions(y) - self._call_mean(self._x), dtype=np.float64)
        if not np.isfinite(c):
            raise ValueError("mean function returned NaN or Inf for parameters:\n{0}".format(
                self.mean.get_parameter_dict(include_frozen=True)))
        y = self._check_dimensions(y)
        if c == 0.0:
            return np.ascontiguousarray(y, dtype=np.float64)  # (no copy when y already is one)
        return np.ascontiguousarray(y - c, dtype=np.float64)

    def _call_white_noise_gradient(self, x):
        return self.white_noise.get_gradient(self._model_input(x))

    # -- state -----------------------------------------------------------------------------------------------------
    @property
    def computed(self):
        """Is the factorisation current w.r.t. the kernel parameters?"""
        return self._computed and self.solver.computed and (self.kernel is None or not self.kernel.dirty)

    @computed.setter
    def computed(self, v):
        self._computed = v
        if v and self.kernel is not None:
            self.kernel.dirty = False

    def parse_samples(self, t):
        """Coerce coordinates to ``(nsamples, ndim)``; 1-D input means one-dimensional samples."""
        t = np.atleast_1d(t)
        if t.ndim == 1:
            t = np.atleast_2d(t).T
        if t.ndim != 2 or (self.kernel is not None and t.shape[1] != self.kernel.ndim):
            raise ValueError("Dimension mismatch")
        return t

    def _check_dimensions(self, y, check_dim=True):
        n = self._x.shape[0]
        y = np.atleast_1d(y)
        if check_dim and y.ndim > 1:
            raise ValueError("The predicted dimension must be 1-D")
        if len(y) != n:
            raise ValueError("Dimension mismatch")
        return y

    def _residual(self, y):
        return np.ascontiguousarray(self._check_dimensions(y) - self._call_mean(self._x), dtype=np.float64)

    def _compute_alpha(self, y, cache):
        """alpha = K^-1 (y - mean); cached on the identity of y's values (gp.py:260-275)."""
        if not cache:
            return self.solver.apply_inverse(self._residual(y), in_place=True).flatten()
        if self._alpha is None or not np.array_equiv(y, self._y):
            self._y = y
            self._alpha = self.solver.apply_inverse(self._residual(y), in_place=True).flatten()
        return self._alpha

    def apply_inverse(self, y):
        """``K^-1 (y - mean)`` for a vector or an ``(nsamples, K)`` matrix."""
        self.recompute(quiet=False)
        r = np.array(y, dtype=np.float64, order="F")
        r = self._check_dimensions(r, check_dim=False)
        mu = self._call_mean(self._x)
        r -= mu.reshape((-1,) + (1,) * (r.ndim - 1))
        b = self.solver.apply_inverse(r, in_place=True)
        return b.flatten() if r.ndim == 1 else b

    # -- the hot path ------------------------------------------------------------------------------------------------
    def compute(self, x, yerr=0.0, **kwargs):
        """Build and factorise the covariance matrix for coordinates ``x`` and uncertainties ``yerr``."""
        self._x = np.ascontiguousarray(self.parse_samples(x), dtype=np.float64)
        try:
            self._yerr2 = float(yerr) ** 2 * np.ones(len(x))
        except TypeError:
            self._yerr2 = self._check_dimensions(yerr) ** 2
        self._yerr2 = np.ascontiguousarray(self._yerr2, dtype=np.float64)

        # a new solver per compute: the factorisation is a snapshot of the current parameters
        self.solver = self.solver_type(self.kernel, **(self.solver_kwargs))
        self.solver.compute(self._x, self._sigma(self._x), **kwargs)

        self._const = -0.5 * (len(self._x) * np.log(2 * np.pi) + self.solver.log_determinant)
        self.computed = True
        self._alpha = None

    def recompute(self, quiet=False, **kwargs):
        """Refactorise if the kernel changed since the last ``compute``.  With ``quiet`` a failed factorisation
        returns ``False`` instead of raising."""
        if self.computed:
            return True
        if not (hasattr(self, "_x") and hasattr(self, "_yerr2")):
            raise RuntimeError("You need to compute the model first")
        try:
            self.compute(self._x, np.sqrt(self._yerr2), **kwargs)
        except (ValueError, LinAlgError):
            if quiet:
                return False
            raise
        return True

    def log_likelihood(self, y, quiet=False):
        """Marginal log-likelihood of ``y`` at the computed coordinates; ``-inf`` on failure when ``quiet``."""
        if not self.recompute(quiet=quiet):
            return -np.inf
        try:
            r = self._residual_of(y)
        except ValueError as exc:
            if quiet and "mean function" in str(exc):
                return -np.inf
            raise
        ll = self._const - 0.5 * self.solver.dot_solve(r)
        return ll if np.isfinite(ll) else -np.inf

    def batch_log_likelihood(self, vectors, y, quiet=False):
        """:func:`log_likelihood` at many parameter vectors: entry ``b`` of the ``(B,)`` result is what
        ``gp.set_parameter_vector(vectors[b]); gp.log_likelihood(y, quiet=quiet)`` returns on the computed ``x`` and
        ``yerr`` (an ensemble sampler's ``vectorize=True`` step).  With ``quiet`` a failing member is ``-inf`` and the
        others are unaffected; otherwise the exception that loop raises first is raised.  The GP is left as it was:
        parameter vector, factorisation, cached solve and dirty flags.

        Solvers with a ``batch_log_likelihood`` hook (``BasicSolver``) factorise all members in one batched pass on
        the device; any other solver (``HODLRSolver``, ``TrivialSolver``, plug-ins) runs that loop.

        :param vectors: ``(B, len(gp))`` active-parameter vectors, as :func:`set_parameter_vector` takes them
        """
        if not (hasattr(self, "_x") and hasattr(self, "_yerr2")):
            raise RuntimeError("You need to compute the model first")
        vectors = np.asarray(vectors, dtype=np.float64)
        if vectors.ndim != 2 or vectors.shape[1] != len(self):
            raise ValueError("vectors must have shape (B, {0}), got {1}".format(len(self), vectors.shape))
        if vectors.shape[0] == 0:
            return np.empty(0, dtype=np.float64)
        batch = getattr(self.solver_type, "batch_log_likelihood", None)
        if batch is not None:
            out = self._batch_device(batch, vectors, y, quiet)
            if out is not None:
                return out
        return self._batch_loop(vectors, y, quiet)

    def _batch_state(self):
        return (self.get_parameter_vector(include_frozen=True), [m.dirty for m in self.models.values()],
                dict((k, self.__dict__[k]) for k in ("_computed", "solver", "_alpha", "_y", "_const", "_x", "_yerr2")
                     if k in self.__dict__))

    def _batch_restore(self, state):
        vector, dirty, attrs = state
        self.set_parameter_vector(vector, include_frozen=True)
        for m, d in zip(self.models.values(), dirty):
            m.dirty = d
        self.__dict__.update(attrs)

    def _batch_loop(self, vectors, y, quiet):
        state = self._batch_state()
        try:
            out = np.empty(len(vectors), dtype=np.float64)
            for b, v in enumerate(vectors):
                self.set_parameter_vector(v)
                out[b] = self.log_likelihood(y, quiet=quiet)
            return out
        finally:
            self._batch_restore(state)

    def _swap_eval(self, model, vector, fn):
        """``fn()`` with only ``model``'s full parameter vector set to ``vector``; the model is restored after."""
        saved, dirty = model.get_parameter_vector(include_frozen=True), model.dirty
        try:
            model.set_parameter_vector(vector, include_frozen=True)
            return fn()
        finally:
            model.set_parameter_vector(saved, include_frozen=True)
            model.dirty = dirty

    def _batch_members(self, vectors, y, residual, const_residual):
        """The per-member host inputs of the batched dense paths: ``(spec, full, kpar, sigma, resid, fact_err,
        mean_err)``, or ``None`` when the kernel has no valid device program (the loop then reproduces whatever the
        per-vector path does with it).  ``full`` holds the members' full parameter vectors, ``kpar`` their kernel part;
        ``sigma`` and ``resid`` (``(B, n)``) are built with the elementwise operations of :func:`_sigma` and of
        ``residual`` (the method the single path forms its residual with), ``const_residual(c)`` being that residual
        for a constant mean ``c``.  ``fact_err[b]`` / ``mean_err[b]`` is the exception the per-vector path meets while
        factorising (white noise) and while forming the residual (mean), or ``None``."""
        try:
            spec = flatten(self.kernel)
        except Exception:
            return None
        if _lib.load().bgp_spec_validate(C.byref(spec)) != _lib.BGP_OK:
            return None
        nb, n = len(vectors), len(self._x)
        full = np.tile(self.get_parameter_vector(include_frozen=True), (nb, 1))
        full[:, self.unfrozen_mask] = vectors
        n_mean, n_wn = self.mean.full_size, self.white_noise.full_size
        kpar = np.ascontiguousarray(full[:, n_mean + n_wn:])
        if kpar.shape[1] != num_params(spec):
            return None
        y = self._check_dimensions(y)

        fact_err, mean_err = [None] * nb, [None] * nb
        sigma = np.empty((nb, n), dtype=np.float64)
        if type(self.white_noise) is ConstantModel:
            for b in range(nb):  # the operations of GP._sigma, member by member
                sigma[b] = self._yerr2 + np.exp(float(full[b, n_mean]))
            np.sqrt(sigma, out=sigma)
        else:
            for b in range(nb):
                try:
                    sigma[b] = self._swap_eval(self.white_noise, full[b, n_mean:n_mean + n_wn],
                                               lambda: self._sigma(self._x))
                except Exception as exc:
                    fact_err[b] = exc
                    sigma[b] = 1.0
        resid = np.empty((nb, n), dtype=np.float64)
        if type(self.mean) is ConstantModel:
            for b in range(nb):
                c = float(full[b, 0])
                if not np.isfinite(c):
                    try:
                        self._swap_eval(self.mean, full[b, :n_mean], lambda: residual(y))
                    except Exception as exc:
                        mean_err[b] = exc
                    resid[b] = 0.0
                else:
                    resid[b] = const_residual(y, c)
        else:
            for b in range(nb):
                try:
                    resid[b] = self._swap_eval(self.mean, full[b, :n_mean], lambda: residual(y))
                except Exception as exc:
                    mean_err[b] = exc
                    resid[b] = 0.0
        for b in range(nb):  # the per-vector solve rejects a non-finite right-hand side (BasicSolver, as scipy does)
            if mean_err[b] is None and not np.all(np.isfinite(resid[b])):
                mean_err[b] = ValueError(NONFINITE_RHS)
                resid[b] = 0.0
        return spec, full, kpar, sigma, resid, fact_err, mean_err

    @staticmethod
    def _batch_factor_error(spec, kpar, b, err, info):
        """The exception member ``b``'s factorisation raises on the per-vector path (``err``: the white-noise one),
        from the batch's ``info``; ``None`` when it succeeds."""
        if err is not None or info == 0:
            return err
        if info > 0:
            return LinAlgError("%d-th leading minor of the array is not positive definite" % info)
        member = patch_specs(spec, kpar[b:b + 1])[0]
        try:
            _lib.check(_lib.load().bgp_spec_validate(C.byref(member)))
        except Exception as e:
            return e
        return ValueError("invalid kernel")

    def _batch_device(self, batch, vectors, y, quiet):
        """The batched dense path of :func:`batch_log_likelihood`; ``None`` when the kernel has no valid device
        program."""
        members = self._batch_members(vectors, y, self._residual_of,
                                      lambda y, c: y if c == 0.0 else y - c)  # the operations of GP._residual_of
        if members is None:
            return None
        spec, _, kpar, sigma, resid, fact_err, mean_err = members
        n = len(self._x)
        log_det, quad, info = batch(spec, kpar, self._x, sigma, resid)
        # GP.compute / GP.log_likelihood, in the same order of operations
        const = -0.5 * (n * np.log(2 * np.pi) + log_det)
        ll = const - 0.5 * quad
        ll[~np.isfinite(ll)] = -np.inf
        for b in range(len(vectors)):
            exc = self._batch_factor_error(spec, kpar, b, fact_err[b], info[b])
            if exc is not None:
                ll[b] = -np.inf
                if not (quiet and isinstance(exc, (ValueError, LinAlgError))):
                    raise exc
                continue
            exc = mean_err[b]
            if exc is not None:
                ll[b] = -np.inf
                if not (quiet and isinstance(exc, ValueError) and "mean function" in str(exc)):
                    raise exc
        return ll

    def batch_predict(self, vectors, y, t, return_cov=True, return_var=False, kernel=None):
        """:func:`predict` at many parameter vectors: ``mu`` (``(B, ns)``), ``(mu, var)`` or ``(mu, cov)`` (``var``
        ``(B, ns)``, ``cov`` ``(B, ns, ns)``; ``return_var`` wins, as in :func:`predict`).  Entry ``b`` is bit for bit
        what ``gp.set_parameter_vector(vectors[b]); gp.predict(y, t, return_cov=..., return_var=...)`` returns on the
        computed ``x`` and ``yerr``: the posterior predictive of a sampler's chain in one call.  The GP is left as it
        was: parameter vector, factorisation, cached solve and dirty flags.

        The call raises the exception that loop would raise first, with its type and message, with one difference:
        the checks that do not depend on the member (the shape of ``vectors``, ``y``'s length, ``t``'s dimension)
        come first, so when member 0 would also fail to factorise the loop raises that error instead.  With no
        members or no test points nothing is computed and the empty results are returned.

        Solvers with a ``batch_predict`` hook (``BasicSolver``) factorise and predict all members in one batched pass
        on the device; any other solver (``HODLRSolver``, ``TrivialSolver``, plug-ins), and an explicit ``kernel``,
        take that loop.

        :param vectors: ``(B, len(gp))`` active-parameter vectors, as :func:`set_parameter_vector` takes them
        """
        if not (hasattr(self, "_x") and hasattr(self, "_yerr2")):
            raise RuntimeError("You need to compute the model first")
        vectors = np.asarray(vectors, dtype=np.float64)
        if vectors.ndim != 2 or vectors.shape[1] != len(self):
            raise ValueError("vectors must have shape (B, {0}), got {1}".format(len(self), vectors.shape))
        self._check_dimensions(y)
        xs = self.parse_samples(t)
        what = "var" if return_var else ("cov" if return_cov else None)
        nb, ns = len(vectors), len(xs)
        if nb == 0 or ns == 0:
            mu = np.empty((nb, ns), dtype=np.float64)
            if what is None:
                return mu
            return mu, np.empty((nb, ns) if what == "var" else (nb, ns, ns), dtype=np.float64)
        batch = getattr(self.solver_type, "batch_predict", None)
        if batch is not None and kernel is None:
            out = self._batch_predict_device(batch, vectors, y, xs, what)
            if out is not None:
                return out
        return self._batch_predict_loop(vectors, y, t, return_cov, return_var, kernel)

    def _batch_predict_loop(self, vectors, y, t, return_cov, return_var, kernel):
        state = self._batch_state()
        try:
            res = []
            for v in vectors:
                self.set_parameter_vector(v)
                res.append(self.predict(y, t, return_cov=return_cov, return_var=return_var, kernel=kernel))
        finally:
            self._batch_restore(state)
        if not (return_var or return_cov):
            return np.stack(res)
        return np.stack([r[0] for r in res]), np.stack([r[1] for r in res])

    def _batch_predict_device(self, batch, vectors, y, xs, what):
        """The batched dense path of :func:`batch_predict`; ``None`` when the kernel has no valid device program."""
        members = self._batch_members(vectors, y, self._residual,
                                      lambda y, c: y - (c + np.zeros(len(y))))  # GP._residual of a ConstantModel
        if members is None:
            return None
        spec, full, kpar, sigma, resid, fact_err, mean_err = members
        nb, ns, n_mean = len(vectors), len(xs), self.mean.full_size
        # the mean model at x*, what GP.predict adds last (a non-finite constant already failed in the residual)
        mean_xs, xs_err = np.zeros((nb, ns), dtype=np.float64), [None] * nb
        for b in range(nb):
            if type(self.mean) is ConstantModel:
                mean_xs[b] = float(full[b, 0]) + np.zeros(ns)
                continue
            try:
                mean_xs[b] = self._swap_eval(self.mean, full[b, :n_mean], lambda: self._call_mean(xs))
            except Exception as exc:
                xs_err[b] = exc
        mu, out, info = batch(spec, kpar, self._x, sigma, resid, xs, what)
        for b in range(nb):  # the loop's order: white noise, factorisation, residual, mean at x*
            exc = self._batch_factor_error(spec, kpar, b, fact_err[b], info[b])
            exc = exc if exc is not None else (mean_err[b] if mean_err[b] is not None else xs_err[b])
            if exc is not None:
                raise exc
        mu += mean_xs
        return mu if what is None else (mu, out)

    def lnlikelihood(self, y, quiet=False):
        warnings.warn("'lnlikelihood' is deprecated. Use 'log_likelihood'", DeprecationWarning)
        return self.log_likelihood(y, quiet=quiet)

    def grad_log_likelihood(self, y, quiet=False):
        """Gradient of :func:`log_likelihood` w.r.t. the active parameter vector (gp.py:406-468)."""
        nothing = np.zeros(len(self), dtype=np.float64)
        if not self.recompute(quiet=quiet):
            return nothing
        n_wn, n_k, n_mean = len(self.white_noise), len(self.kernel), len(self.mean)
        fused = getattr(self.solver, "grad_terms", None) if (n_wn or n_k) else None
        try:
            if fused is not None:
                # alpha, the kernel-gradient contraction and diag(alpha alpha^T - K^-1) in one device pass: neither
                # K^-1 nor the (N, N, P) gradient tensor visits the host (reference gp.py:437-466 forms both)
                mask = self.kernel.unfrozen_mask
                terms = fused(self._residual(y), mask.astype(np.uint32))
                if terms is None:
                    fused = None
                else:
                    alpha, gk, diagA = terms
            if fused is None:
                alpha = self._compute_alpha(y, False)
        except ValueError:
            if quiet:
                return nothing
            raise

        if fused is None and (n_wn or n_k):
            A = np.outer(alpha, alpha) - self.solver.get_inverse()
            diagA = np.diag(A)

        grad = np.empty(len(self))
        pos = 0
        if n_mean:
            try:
                dmu = self._call_mean_gradient(self._x)
            except ValueError:
                if quiet:
                    return nothing
                raise
            grad[pos:pos + n_mean] = np.dot(dmu, alpha)
            pos += n_mean
        if n_wn:
            wn = self._call_white_noise(self._x)
            dwn = self._call_white_noise_gradient(self._x)
            grad[pos:pos + n_wn] = 0.5 * np.sum((np.exp(wn) * diagA)[None, :] * dwn, axis=1)
            pos += n_wn
        if n_k:
            if fused is not None:
                grad[pos:pos + n_k] = 0.5 * gk[mask]
            else:
                # plug-in solvers without grad_terms: K^-1 comes from the solver, the contraction still runs on the
                # device without the (N, N, P) tensor
                mask = self.kernel.unfrozen_mask
                grad[pos:pos + n_k] = 0.5 * self.kernel.kernel.gradient_contract(mask.astype(np.uint32), self._x, A)[mask]
        return grad

    def batch_grad_log_likelihood(self, vectors, y, quiet=False, return_log_likelihood=False):
        """:func:`grad_log_likelihood` at many parameter vectors: row ``b`` of the ``(B, len(gp))`` result is bit for
        bit what ``gp.set_parameter_vector(vectors[b]); gp.grad_log_likelihood(y, quiet=quiet)`` returns on the
        computed ``x`` and ``yerr`` (chains of a gradient-based sampler in lock-step, the starts of a multi-start fit).
        With ``return_log_likelihood`` the result is ``(ll, grad)``: ``ll[b]`` is what :func:`log_likelihood` returns
        when that loop calls it before the gradient, bit for bit :func:`batch_log_likelihood`'s, and value and
        gradient come from one factorisation.

        With ``quiet`` a failing member gets the loop's ``-inf`` and zero gradient and the others are unaffected;
        otherwise the exception that loop raises first is raised, with its type and message, with one difference: the
        checks that do not depend on the member (the shape of ``vectors``, ``y``'s length) come first.  The GP is left
        as it was: parameter vector, factorisation, cached solve and dirty flags.

        Solvers with a ``batch_grad_terms`` hook (``BasicSolver``) factorise all members, form their ``K^-1`` and
        contract the kernel gradients in one batched pass on the device.  Any other solver (``HODLRSolver``,
        ``TrivialSolver``, plug-ins) takes that loop, and so do a kernel without a valid device program, one with more
        than 64 parameters (the device contraction's limit: every member's gradient then fails as it does in the
        loop) and a GP whose only active parameters are the mean's.

        :param vectors: ``(B, len(gp))`` active-parameter vectors, as :func:`set_parameter_vector` takes them
        """
        if not (hasattr(self, "_x") and hasattr(self, "_yerr2")):
            raise RuntimeError("You need to compute the model first")
        vectors = np.asarray(vectors, dtype=np.float64)
        if vectors.ndim != 2 or vectors.shape[1] != len(self):
            raise ValueError("vectors must have shape (B, {0}), got {1}".format(len(self), vectors.shape))
        self._check_dimensions(y)
        out = None
        if len(vectors) == 0:
            out = np.empty(0, dtype=np.float64), np.empty((0, len(self)), dtype=np.float64)
        batch = getattr(self.solver_type, "batch_grad_terms", None)
        if out is None and batch is not None and (len(self.white_noise) or len(self.kernel)):
            out = self._batch_grad_device(batch, vectors, y, quiet, return_log_likelihood)
        if out is None:
            out = self._batch_grad_loop(vectors, y, quiet, return_log_likelihood)
        return out if return_log_likelihood else out[1]

    def _batch_grad_loop(self, vectors, y, quiet, return_ll):
        state = self._batch_state()
        try:
            ll = np.empty(len(vectors), dtype=np.float64)
            grad = np.empty((len(vectors), len(self)), dtype=np.float64)
            for b, v in enumerate(vectors):
                self.set_parameter_vector(v)
                if return_ll:
                    ll[b] = self.log_likelihood(y, quiet=quiet)
                grad[b] = self.grad_log_likelihood(y, quiet=quiet)
            return ll, grad
        finally:
            self._batch_restore(state)

    def _batch_grad_device(self, batch, vectors, y, quiet, return_ll):
        """The batched dense path of :func:`batch_grad_log_likelihood`: ``(ll, grad)``, or ``None`` when the kernel
        has no valid device program or more than ``_MAX_GRAD_PARAMS`` parameters."""
        # one residual serves both terms: GP._residual (the gradient's) and GP._residual_of (the value's) round alike
        members = self._batch_members(vectors, y, self._residual,
                                      lambda y, c: y - (c + np.zeros(len(y))))  # GP._residual of a ConstantModel
        if members is None or members[2].shape[1] > _MAX_GRAD_PARAMS:
            return None
        spec, full, kpar, sigma, resid, fact_err, mean_err = members
        nb, n = len(vectors), len(self._x)
        mask = self.kernel.unfrozen_mask
        log_det, quad, alpha, g, diag, info = batch(spec, kpar, self._x, sigma, resid, mask.astype(np.uint32))
        # GP.compute / GP.log_likelihood, in the same order of operations
        const = -0.5 * (n * np.log(2 * np.pi) + log_det)
        ll = const - 0.5 * quad
        ll[~np.isfinite(ll)] = -np.inf
        # GP.grad_log_likelihood member by member, with its operations
        n_mean, n_wn, n_k = len(self.mean), len(self.white_noise), len(self.kernel)
        full_mean, full_wn = self.mean.full_size, self.white_noise.full_size
        grad = np.zeros((nb, len(self)), dtype=np.float64)
        for b in range(nb):  # the loop's order: factorisation (white noise included), residual, mean gradient
            exc = self._batch_factor_error(spec, kpar, b, fact_err[b], info[b])
            if exc is not None:
                if not (quiet and isinstance(exc, (ValueError, LinAlgError))):
                    raise exc
                ll[b] = -np.inf
                continue
            exc = mean_err[b]
            if exc is not None:
                # log_likelihood swallows only the mean's own ValueError under quiet, grad_log_likelihood any ValueError
                if not (quiet and isinstance(exc, ValueError) and (not return_ll or "mean function" in str(exc))):
                    raise exc
                ll[b] = -np.inf
                continue
            pos = 0
            if n_mean:
                try:
                    dmu = self._swap_eval(self.mean, full[b, :full_mean], lambda: self._call_mean_gradient(self._x))
                except ValueError:
                    if quiet:
                        continue
                    raise
                grad[b, pos:pos + n_mean] = np.dot(dmu, alpha[b])
                pos += n_mean
            if n_wn:
                wn, dwn = self._swap_eval(self.white_noise, full[b, full_mean:full_mean + full_wn],
                                          lambda: (self._call_white_noise(self._x),
                                                   self._call_white_noise_gradient(self._x)))
                grad[b, pos:pos + n_wn] = 0.5 * np.sum((np.exp(wn) * diag[b])[None, :] * dwn, axis=1)
                pos += n_wn
            if n_k:
                grad[b, pos:pos + n_k] = 0.5 * g[b][mask]
        return ll, grad

    def grad_lnlikelihood(self, y, quiet=False):
        warnings.warn("'grad_lnlikelihood' is deprecated. Use 'grad_log_likelihood'", DeprecationWarning)
        return self.grad_log_likelihood(y, quiet=quiet)

    def nll(self, vector, y, quiet=True):
        self.set_parameter_vector(vector)
        if not np.isfinite(self.log_prior()):
            return np.inf
        return -self.log_likelihood(y, quiet=quiet)

    def grad_nll(self, vector, y, quiet=True):
        self.set_parameter_vector(vector)
        if not np.isfinite(self.log_prior()):
            return np.zeros(len(vector))
        return -self.grad_log_likelihood(y, quiet=quiet)

    def predict(self, y, t, return_cov=True, return_var=False, cache=True, kernel=None):
        """Conditional predictive distribution at ``t``: ``mu``, ``(mu, cov)`` or ``(mu, var)``."""
        self.recompute()
        alpha = self._compute_alpha(y, cache)
        xs = self.parse_samples(t)
        if kernel is None:
            kernel = self.kernel

        if not (return_var or return_cov):
            # mean only: K(x*, x) alpha evaluated matrix-free on the device (csrc/kmat_ops.cu); the reference forms the
            # (n*, N) matrix on the host (gp.py:524-528), which stops being possible long before N = 2^18
            return kernel.matvec(xs, self._x, alpha) + self._call_mean(xs)

        # variance / covariance from the stored factorisation on the device (BasicSolver, HODLRSolver): K(x*, x) and
        # K^-1 K(x, x*) stay there, streamed in column chunks.  Solvers without `predictive`, or that return None (a
        # pickled dense factor, a sharded tree), take the reference's host route below.
        predictive = getattr(self.solver, "predictive", None)
        out = predictive(kernel, xs, "var" if return_var else "cov") if predictive is not None else None
        if out is not None:
            return kernel.matvec(xs, self._x, alpha) + self._call_mean(xs), out
        return self._predict_host(alpha, xs, return_var, kernel)

    def _predict_host(self, alpha, xs, return_var, kernel):
        """The reference's route (gp.py:534-545): K(x*, x) on the host, ``solver.apply_inverse`` on its transpose."""
        Kxs = kernel.get_value(xs, self._x)
        mu = np.dot(Kxs, alpha) + self._call_mean(xs)

        KinvKxs = self.solver.apply_inverse(Kxs.T)
        if return_var:
            var = kernel.get_value(xs, diag=True)
            var -= np.sum(Kxs.T * KinvKxs, axis=0)
            return mu, var
        cov = kernel.get_value(xs)
        cov -= np.dot(Kxs, KinvKxs)
        return mu, cov

    def sample_conditional(self, y, t, size=1):
        mu, cov = self.predict(y, t)
        return multivariate_gaussian_samples(cov, size, mean=mu)

    def sample(self, t=None, size=1):
        """Draw from the prior, at ``t`` or (``t is None``) at the computed coordinates via the Cholesky factor."""
        if t is None:
            self.recompute()
            n = self._x.shape[0]
            draws = self.solver.apply_sqrt(np.random.randn(size, n))
            draws += self._call_mean(self._x)
            return draws[0] if size == 1 else draws
        x = self.parse_samples(t)
        cov = self.get_matrix(x)
        cov[np.diag_indices_from(cov)] += TINY
        return multivariate_gaussian_samples(cov, size, mean=self._call_mean(x))

    def get_matrix(self, x1, x2=None):
        x1 = self.parse_samples(x1)
        if x2 is None:
            return self.kernel.get_value(x1)
        return self.kernel.get_value(x1, self.parse_samples(x2))

    # modeling-protocol synonyms
    def get_value(self, *args, **kwargs):
        return self.log_likelihood(*args, **kwargs)

    def get_gradient(self, *args, **kwargs):
        return self.grad_log_likelihood(*args, **kwargs)
