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
from ._spec import BGP_MAX_DIM, flatten, num_params, patch_specs
from .modeling import ConstantModel, ModelSet
from .parallel import ShardedHODLRSolver
from .solvers import BasicSolver, HODLRSolver, TrivialSolver
from .solvers.basic import NONFINITE_RHS, _check_finite
from .solvers.hodlr import FISHER_HODLR
from .utils import device_gaussian_samples, multivariate_gaussian_samples

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


def _check_rng(rng):
    if not isinstance(rng, (np.random.Generator, np.random.RandomState)):
        raise TypeError("rng must be a numpy.random.Generator or numpy.random.RandomState, got {0}".format(
            type(rng).__name__))


def _sampling_jitter(rng, jitter):
    """The ``rng`` / ``jitter`` checks of the conditional draws: the jitter the device draws add (``TINY`` by
    default), ``None`` without ``rng``, where no jitter may be given."""
    if rng is None:
        if jitter is not None:
            raise ValueError("jitter applies only to draws with an rng; the host route adds nothing")
        return None
    _check_rng(rng)
    jitter = TINY if jitter is None else float(jitter)
    if not (np.isfinite(jitter) and jitter >= 0.0):
        raise ValueError("jitter must be finite and >= 0, got {0}".format(jitter))
    return jitter


def _check_grad_predict_mean(mean, method="grad_predict", model="mean"):
    if type(mean) is not ConstantModel:
        raise NotImplementedError("{0} needs the {1} model's gradient with respect to the inputs, which the modeling "
                                  "protocol does not provide; only a constant {1} is supported".format(method, model))


def _check_grad_predict_dim(xs):
    if xs.shape[1] > BGP_MAX_DIM:
        raise ValueError("input-coordinate gradients support at most {0} dimensions (got {1})".format(
            BGP_MAX_DIM, xs.shape[1]))


def _check_size(size):
    size = int(size)
    if size < 0:
        raise ValueError("size must be >= 0, got {0}".format(size))
    return size


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

    def _require_computed(self):
        if not (hasattr(self, "_x") and hasattr(self, "_yerr2")):
            raise RuntimeError("You need to compute the model first")

    def recompute(self, quiet=False, **kwargs):
        """Refactorise if the kernel changed since the last ``compute``.  With ``quiet`` a failed factorisation
        returns ``False`` instead of raising."""
        if self.computed:
            return True
        self._require_computed()
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
        vectors = self._batch_vectors(vectors)
        if vectors.shape[0] == 0:
            return np.empty(0, dtype=np.float64)
        batch = getattr(self.solver_type, "batch_log_likelihood", None)
        if batch is not None:
            out = self._batch_device(batch, vectors, y, quiet)
            if out is not None:
                return out
        return np.array(self._batch_loop(vectors, lambda: self.log_likelihood(y, quiet=quiet)), dtype=np.float64)

    def _batch_vectors(self, vectors):
        """The checks of every ``batch_*`` method that come before its own: a computed model and ``vectors`` of shape
        ``(B, len(gp))``, returned as a float64 array."""
        self._require_computed()
        vectors = np.asarray(vectors, dtype=np.float64)
        if vectors.ndim != 2 or vectors.shape[1] != len(self):
            raise ValueError("vectors must have shape (B, {0}), got {1}".format(len(self), vectors.shape))
        return vectors

    def _batch_loop(self, vectors, fn):
        """The per-vector path of the ``batch_*`` methods: ``[fn() for each member]`` with ``set_parameter_vector``
        called for the member before ``fn``.  The GP is left as it was: parameter vector, factorisation, cached solve
        and dirty flags."""
        vector, dirty = self.get_parameter_vector(include_frozen=True), [m.dirty for m in self.models.values()]
        attrs = dict((k, self.__dict__[k]) for k in ("_computed", "solver", "_alpha", "_y", "_const", "_x", "_yerr2")
                     if k in self.__dict__)
        try:
            res = []
            for v in vectors:
                self.set_parameter_vector(v)
                res.append(fn())
            return res
        finally:
            self.set_parameter_vector(vector, include_frozen=True)
            for m, d in zip(self.models.values(), dirty):
                m.dirty = d
            self.__dict__.update(attrs)

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
        factorising (white noise) and while forming the residual (mean), or ``None``.  With ``y`` ``None`` no residual
        is formed: ``resid`` is ``None`` and ``mean_err`` all ``None``."""
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
        if y is not None:
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
        if y is None:
            return spec, full, kpar, sigma, None, fact_err, mean_err
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
    def _member_error(spec, kpar, b, info, fact_err, *later):
        """The exception member ``b`` meets first on the per-vector path, or ``None``: the white noise
        (``fact_err[b]``) or the factorisation (from the batch's ``info[b]``), then the first of ``later`` (per-member
        lists of an exception or ``None``, in the loop's order)."""
        exc = fact_err[b]
        if exc is None and info[b] > 0:
            exc = LinAlgError("%d-th leading minor of the array is not positive definite" % info[b])
        elif exc is None and info[b] < 0:
            member = patch_specs(spec, kpar[b:b + 1])[0]
            try:
                _lib.check(_lib.load().bgp_spec_validate(C.byref(member)))
            except Exception as e:
                exc = e
            else:
                exc = ValueError("invalid kernel")
        for errs in later:
            if exc is None:
                exc = errs[b]
        return exc

    def _raise_member_error(self, spec, kpar, info, fact_err, *later):
        """Raise the exception the per-vector loop meets first, member by member (:func:`_member_error`)."""
        for b in range(len(info)):
            exc = self._member_error(spec, kpar, b, info, fact_err, *later)
            if exc is not None:
                raise exc

    def _member_failed(self, spec, kpar, b, info, fact_err, mean_err, quiet, any_value_error):
        """Whether member ``b`` fails in the white noise, the factorisation or the residual, the first stages of the
        value and gradient paths.  The failure is raised unless ``quiet`` absorbs it as the single calls do: a
        ``ValueError`` or ``LinAlgError`` of the white noise or the factorisation (``recompute``), and a ``ValueError``
        of the residual, any one when ``any_value_error`` (the gradients) or only the mean function's own (the values,
        which let the solver's non-finite right-hand side through)."""
        exc = self._member_error(spec, kpar, b, info, fact_err)
        if exc is not None:
            absorbed = quiet and isinstance(exc, (ValueError, LinAlgError))
        else:
            exc = mean_err[b]
            if exc is None:
                return False
            absorbed = quiet and isinstance(exc, ValueError) and (any_value_error or "mean function" in str(exc))
        if absorbed:
            return True
        raise exc

    def _batch_ll(self, log_det, quad):
        """GP.compute / GP.log_likelihood over the members, in the same order of operations."""
        const = -0.5 * (len(self._x) * np.log(2 * np.pi) + log_det)
        ll = const - 0.5 * quad
        ll[~np.isfinite(ll)] = -np.inf
        return ll

    def _batch_device(self, batch, vectors, y, quiet):
        """The batched dense path of :func:`batch_log_likelihood`; ``None`` when the kernel has no valid device
        program."""
        members = self._batch_members(vectors, y, self._residual_of,
                                      lambda y, c: y if c == 0.0 else y - c)  # the operations of GP._residual_of
        if members is None:
            return None
        spec, _, kpar, sigma, resid, fact_err, mean_err = members
        log_det, quad, info = batch(spec, kpar, self._x, sigma, resid)
        ll = self._batch_ll(log_det, quad)
        for b in range(len(vectors)):
            if self._member_failed(spec, kpar, b, info, fact_err, mean_err, quiet, False):
                ll[b] = -np.inf
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
        vectors = self._batch_vectors(vectors)
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
        res = self._batch_loop(vectors, lambda: self.predict(y, t, return_cov=return_cov, return_var=return_var,
                                                             kernel=kernel))
        if not (return_var or return_cov):
            return np.stack(res)
        return np.stack([r[0] for r in res]), np.stack([r[1] for r in res])

    def _batch_predict_device(self, batch, vectors, y, xs, what):
        """The batched dense path of :func:`batch_predict`; ``None`` when the kernel has no valid device program."""
        members = self._batch_predict_members(vectors, y)
        if members is None:
            return None
        spec, full, kpar, sigma, resid, fact_err, mean_err = members
        mean_xs, xs_err = self._batch_mean_at(full, xs)
        mu, out, info = batch(spec, kpar, self._x, sigma, resid, xs, what)
        self._raise_member_error(spec, kpar, info, fact_err, mean_err, xs_err)  # residual, mean at x*
        mu += mean_xs
        return mu if what is None else (mu, out)

    def _batch_predict_members(self, vectors, y):
        """:func:`_batch_members` with the residual of :func:`predict` (``GP._residual``)."""
        return self._batch_members(vectors, y, self._residual,
                                   lambda y, c: y - (c + np.zeros(len(y))))  # GP._residual of a ConstantModel

    def _batch_mean_at(self, full, xs):
        """``(mean_xs, xs_err)``: the mean model at ``xs`` for each member's full parameter vector (``(B, ns)``), what
        ``GP.predict`` adds last to the kernel part of its mean, and the exception member ``b``'s evaluation raised,
        or ``None`` (a non-finite constant already failed in the residual)."""
        nb, ns, n_mean = len(full), len(xs), self.mean.full_size
        mean_xs, xs_err = np.zeros((nb, ns), dtype=np.float64), [None] * nb
        for b in range(nb):
            if type(self.mean) is ConstantModel:
                mean_xs[b] = float(full[b, 0]) + np.zeros(ns)
                continue
            try:
                mean_xs[b] = self._swap_eval(self.mean, full[b, :n_mean], lambda: self._call_mean(xs))
            except Exception as exc:
                xs_err[b] = exc
        return mean_xs, xs_err

    def lnlikelihood(self, y, quiet=False):
        warnings.warn("'lnlikelihood' is deprecated. Use 'log_likelihood'", DeprecationWarning)
        return self.log_likelihood(y, quiet=quiet)

    def grad_log_likelihood(self, y, quiet=False):
        """Gradient of :func:`log_likelihood` w.r.t. the active parameter vector (gp.py:406-468)."""
        nothing = np.zeros(len(self), dtype=np.float64)
        if not self.recompute(quiet=quiet):
            return nothing
        layout = n_mean, n_wn, n_k = self._grad_layout()
        mask = self.kernel.unfrozen_mask
        gk = diagA = dmu = None
        fused = getattr(self.solver, "grad_terms", None) if (n_wn or n_k) else None
        try:
            if fused is not None:
                # alpha, the kernel-gradient contraction and diag(alpha alpha^T - K^-1) in one device pass: neither
                # K^-1 nor the (N, N, P) gradient tensor visits the host (reference gp.py:437-466 forms both)
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
        if n_mean:
            try:
                dmu = self._call_mean_gradient(self._x)
            except ValueError:
                if quiet:
                    return nothing
                raise
        if fused is None and n_k:
            # plug-in solvers without grad_terms: K^-1 comes from the solver, the contraction still runs on the
            # device without the (N, N, P) tensor
            gk = self.kernel.kernel.gradient_contract(mask.astype(np.uint32), self._x, A)
        return self._grad_row(np.empty(len(self)), layout, dmu, alpha, self._white_noise_terms, diagA, gk, mask, 0.5)

    def _white_noise_terms(self):
        """``(wn, dwn)``: the white-noise model and its gradient at the computed coordinates."""
        return self._call_white_noise(self._x), self._call_white_noise_gradient(self._x)

    def _grad_layout(self):
        """``(n_mean, n_wn, n_k)``, the active parameters of each part of a gradient; once per call, outside the
        batches' member loops, as a kernel's size takes tens of microseconds to count."""
        return len(self.mean), len(self.white_noise), len(self.kernel)

    def _grad_row(self, grad, layout, dmu, w, noise, diagA, gk, mask, scale):
        """Fill and return ``grad`` (``(len(gp),)``) in :func:`grad_log_likelihood`'s layout (mean, white noise,
        kernel; frozen parameters left out, ``layout`` from :func:`_grad_layout`): ``dmu . w``,
        ``scale * sum_i exp(wn_i) diagA_i dwn_i`` and ``scale * gk[mask]``, with ``(wn, dwn) = noise()`` called only
        when white-noise parameters are active.  ``scale`` is 1/2 for the marginal likelihood and 1 for the
        leave-one-out log-likelihood (``1.0 * x`` is ``x`` bit for bit)."""
        n_mean, n_wn, n_k = layout
        pos = 0
        if n_mean:
            grad[pos:pos + n_mean] = np.dot(dmu, w)
            pos += n_mean
        if n_wn:
            wn, dwn = noise()
            grad[pos:pos + n_wn] = np.sum((np.exp(wn) * diagA)[None, :] * dwn, axis=1)
            pos += n_wn
        if n_k:
            grad[pos:pos + n_k] = gk[mask]
        grad[n_mean:] *= scale
        return grad

    def _member_gradients(self, layout, full):
        """The mean gradient (``None`` without active mean parameters) of the member whose full parameter vector is
        ``full``, and the ``noise`` of :func:`_grad_row` for that member; both evaluate the models with ``full`` set."""
        n_mean, n_wn = self.mean.full_size, self.white_noise.full_size
        dmu = None
        if layout[0]:
            dmu = self._swap_eval(self.mean, full[:n_mean], lambda: self._call_mean_gradient(self._x))
        return dmu, lambda: self._swap_eval(self.white_noise, full[n_mean:n_mean + n_wn], self._white_noise_terms)

    def grad_log_likelihood_x(self, y, quiet=False, return_gradient=False):
        """Gradient of :func:`log_likelihood` with respect to the training inputs: ``dx[i, q] = d log_likelihood(y) /
        d x[i, q]`` at the computed coordinates, of shape ``(N, ndim)`` (also for 1-D input).  With
        ``return_gradient`` the result is ``(grad, dx)``, ``grad`` from the same pass and the same launches as
        :func:`grad_log_likelihood`: its bits wherever that method is reproducible (dense; HODLR up to N = 1024, whose
        solve adds with atomics above).  This is what fits any parameter that enters through the coordinates, by the chain rule: a
        time delay between two light curves, a warping or drift of one input axis, latent inputs.

        With ``A = alpha alpha^T - K^-1``, ``dx_i = sum_j A_ij d k(x_i, x_j) / d x_i``, the true derivative for every
        metric (each ``x_i`` enters row i and column i of ``K``; the 1/2 of the log-likelihood cancels the factor 2).
        ``yerr`` is data and contributes nothing.  The mean and the white-noise model must be ``ConstantModel`` s (fitted
        or not); anything else raises ``NotImplementedError``, as inputs of more than 8 dimensions raise ``ValueError``,
        before any device work.  ``quiet`` follows :func:`grad_log_likelihood`: a failure it absorbs gives zeros for
        ``dx`` (and ``grad``).

        Solvers with a ``grad_x_terms`` hook (``BasicSolver``, ``HODLRSolver``, ``ShardedHODLRSolver``, collective)
        contract on the device; the HODLR solvers stream ``K^-1`` in column slabs above N = 65536 and contract the input
        gradient in the same pass as the hyper-parameter gradient.  Like their :func:`grad_log_likelihood`, the HODLR
        solvers return the hybrid of ``K~^-1`` (the inverse of the HODLR matrix) with the exact kernel derivative.  Any
        other solver (``TrivialSolver``, plug-ins, a dense solver restored from a pickle) forms ``A`` on the host from
        ``solver.get_inverse()`` and contracts it on the device with ``KernelInterface.x1_gradient_matvec``.
        """
        _check_grad_predict_mean(self.mean, "grad_log_likelihood_x")
        _check_grad_predict_mean(self.white_noise, "grad_log_likelihood_x", "white-noise")
        self._require_computed()
        _check_grad_predict_dim(self._x)
        n, nd = self._x.shape
        fail = (np.zeros(len(self), dtype=np.float64), np.zeros((n, nd), dtype=np.float64))
        if not return_gradient:
            fail = fail[1]
        if not self.recompute(quiet=quiet):
            return fail
        layout = n_mean, n_wn, n_k = self._grad_layout()
        mask = self.kernel.unfrozen_mask
        # grad_log_likelihood's route for each part of grad: the fused terms when white-noise or kernel parameters
        # are active, otherwise alpha from the solve alone
        fused = return_gradient and bool(n_wn or n_k)
        hook = getattr(self.solver, "grad_x_terms", None)
        terms = gk = diagA = dmu = None
        try:
            r = self._residual(y)
            if hook is not None:
                terms = hook(r, mask.astype(np.uint32) if fused else None)
            if terms is None:
                alpha = self._compute_alpha(y, False)
                A = np.outer(alpha, alpha) - self.solver.get_inverse()
                diagA = np.diag(A)
                if fused and n_k:
                    gk = self.kernel.kernel.gradient_contract(mask.astype(np.uint32), self._x, A)
                dx = self.kernel.kernel.x1_gradient_matvec(self._x, self._x, A, scale=1.0)
            else:
                alpha, gk, diagA, dx = terms
            if return_gradient and not fused:
                alpha = self._compute_alpha(y, False)
            if return_gradient and n_mean:
                dmu = self._call_mean_gradient(self._x)
        except ValueError:
            if quiet:
                return fail
            raise
        if not return_gradient:
            return dx
        grad = self._grad_row(np.empty(len(self)), layout, dmu, alpha, self._white_noise_terms, diagA, gk, mask, 0.5)
        return grad, dx

    # -- second order ------------------------------------------------------------------------------------------------
    def fisher_information(self, y=None, quiet=False):
        """The expected Fisher information of the active parameter vector, ``F`` of shape ``(len(gp), len(gp))`` in
        :func:`grad_log_likelihood`'s layout (mean, white noise, kernel; frozen parameters left out; kernel parameters
        in the log units of :func:`get_parameter_vector`):

            F_pq = dmu_p^T K^-1 dmu_q + 1/2 tr(K^-1 dK_p K^-1 dK_q)

        with ``dK = diag(exp(wn) dwn)`` for a white-noise parameter, and zero between mean and covariance parameters.
        It needs first derivatives only, does not depend on ``y`` and is positive semi-definite by construction, so
        after a fit ``inv(F)`` gives the parameters' Cramér-Rao / Laplace covariance (their standard errors), a
        sampler's mass matrix or start ball, and ``p + solve(F, grad)`` a Fisher-scoring step.  ``F`` is exactly
        symmetric, and two calls return the same bits.

        With ``y`` the result is ``(grad, F)``: ``grad`` comes from the same pass and, on ``BasicSolver``, is bit for bit
        :func:`grad_log_likelihood`, so a scoring step costs one ``K^-1``.  ``quiet`` follows
        :func:`grad_log_likelihood`: a failure it absorbs (a failed factorisation, a model returning NaN, more than 64
        kernel parameters) gives zeros for ``F`` (and ``grad``).

        ``BasicSolver`` forms ``K^-1 dK_p K^-1`` for each kernel and white-noise parameter on the FP64 tensor pipe from
        the resident ``K^-1`` (``include/bgp.h: bgp_dense_fisher_terms``), in device memory that does not grow with
        the number of parameters.  ``TrivialSolver``, plug-ins and a dense solver restored from a pickle compute the
        formula on the host from ``solver.apply_inverse(eye(N))`` and ``kernel.get_gradient``.  ``HODLRSolver`` and
        ``ShardedHODLRSolver`` raise ``NotImplementedError`` before any device work.
        """
        self._check_fisher_solver()
        size = len(self)
        fail = np.zeros((size, size), dtype=np.float64)
        if y is not None:
            fail = (np.zeros(size, dtype=np.float64), fail)
        if not self.recompute(quiet=quiet):
            return fail
        layout = n_mean, n_wn, n_k = self._grad_layout()
        mask = self.kernel.unfrozen_mask
        # grad_log_likelihood's route for alpha: the fused terms when white-noise or kernel parameters are active
        fused = y is not None and bool(n_wn or n_k)
        noise = dmu = kinv_dmu = gk = diagA = alpha = None
        try:
            r = self._residual(y) if fused else None
            v = np.zeros((0, len(self._x)), dtype=np.float64)
            if n_wn:
                noise = self._white_noise_terms()
                v = np.exp(noise[0])[None, :] * noise[1]
            rows = rdiag = None
            if n_wn or n_k:
                hook = getattr(self.solver, "fisher_terms", None)
                terms = None if hook is None else hook(r, mask.astype(np.uint32), v)
                if terms is None:
                    rows, rdiag = self._fisher_rows_host(v, n_k)
                    if fused:
                        alpha = self._compute_alpha(y, False)
                        A = np.outer(alpha, alpha) - self.solver.get_inverse()
                        diagA = np.diag(A)
                        if n_k:
                            gk = self.kernel.kernel.gradient_contract(mask.astype(np.uint32), self._x, A)
                else:
                    gterms, rows, rdiag = terms
                    rows = rows[:, mask]
                    if fused:
                        alpha, gk, diagA = gterms
            if y is not None and not fused:
                alpha = self._compute_alpha(y, False)
            if n_mean:
                dmu = self._call_mean_gradient(self._x)
                kinv_dmu = np.asarray(self.solver.apply_inverse(np.array(dmu.T, dtype=np.float64, order="F")),
                                      dtype=np.float64).reshape(len(self._x), n_mean)
        except ValueError:
            if quiet:
                return fail
            raise
        F = self._fisher_matrix(np.zeros((size, size), dtype=np.float64), layout, dmu, kinv_dmu, rows, rdiag, v)
        if y is None:
            return F
        grad = self._grad_row(np.empty(size), layout, dmu, alpha, lambda: noise, diagA, gk, mask, 0.5)
        return grad, F

    def _check_fisher_solver(self):
        """The Fisher information's first check: ``NotImplementedError`` on a HODLR-typed GP, before any work."""
        if isinstance(self.solver_type, type) and issubclass(self.solver_type, (HODLRSolver, ShardedHODLRSolver)):
            raise NotImplementedError(FISHER_HODLR)

    @staticmethod
    def _fisher_matrix(F, layout, dmu, kinv_dmu, rows, rdiag, v):
        """Fill and return the zeroed ``F`` (``(len(gp), len(gp))``) of :func:`fisher_information` from its blocks, for
        the single and the batched paths alike: the mean block ``1/2 (M + M^T)`` with ``M = dmu . K^-1 dmu^T``
        (``kinv_dmu``, ``(N, n_mean)``), and the covariance block ``1/2 (R + R^T)`` with ``R`` the white-noise dots
        ``1/2 rdiag . v^T`` and the kernel entries ``1/2 rows`` (active kernel columns only), ``rows`` and ``rdiag``
        in the solver's row order (kernel, then white noise) and ``v`` the white-noise vectors (``(n_wn, N)``)."""
        n_mean, n_wn, n_k = layout
        if n_mean:
            M = np.dot(dmu, kinv_dmu)
            F[:n_mean, :n_mean] = 0.5 * (M + M.T)
        if n_wn or n_k:
            # R in F's order (white noise, then kernel) from the rows in the solver's order (kernel, then white noise)
            order = np.concatenate([np.arange(n_k, n_k + n_wn), np.arange(n_k)])
            R = np.empty((n_wn + n_k, n_wn + n_k), dtype=np.float64)
            R[:, :n_wn] = 0.5 * np.dot(rdiag[order], v.T)
            R[:, n_wn:] = 0.5 * rows[order]
            F[n_mean:, n_mean:] = 0.5 * (R + R.T)
        return F

    def batch_fisher_information(self, vectors, y=None, quiet=False):
        """:func:`fisher_information` at many parameter vectors: ``F`` of shape ``(B, len(gp), len(gp))``, or with ``y``
        ``(grad, F)`` with ``grad`` ``(B, len(gp))``.  Member ``b`` is bit for bit what
        ``gp.set_parameter_vector(vectors[b]); gp.fisher_information(y, quiet=quiet)`` returns on the computed ``x`` and
        ``yerr``: a Jeffreys prior ``1/2 log det F`` for every walker of an ensemble sampler's step, the metric of
        Riemannian-manifold HMC chains in lock-step, or the Laplace standard errors and Fisher-scoring steps of every
        start of a multi-start fit, in one call.

        With ``quiet`` a failing member gets the loop's zeros and the others are unaffected; otherwise the exception
        that loop raises first is raised, with its type and message (white noise or factorisation, then the residual,
        then the white-noise terms, then the mean gradient), with one difference: the checks that do not depend on the
        member (the shape of ``vectors``, ``y``'s length) come first.  The GP is left as it was: parameter vector,
        factorisation, cached solve and dirty flags.  A HODLR-typed GP raises ``NotImplementedError`` before any work,
        as :func:`fisher_information` does.

        Solvers with a ``batch_fisher_terms`` hook (``BasicSolver``) factorise all members, form their ``K^-1`` and
        every row's ``K^-1 dK K^-1`` in one batched pass on the device, each launch covering all the members of a chunk
        (``include/bgp.h: bgp_dense_batch_fisher_terms``).  Any other solver (``TrivialSolver``, plug-ins) takes that
        loop, and so do a kernel without a valid device program, one with more than 64 parameters (every member then
        fails as it does in the loop) and a GP whose only active parameters are the mean's.

        :param vectors: ``(B, len(gp))`` active-parameter vectors, as :func:`set_parameter_vector` takes them
        """
        self._check_fisher_solver()
        vectors = self._batch_vectors(vectors)
        if y is not None:
            self._check_dimensions(y)
        size = len(self)
        out = None
        if len(vectors) == 0:
            out = np.empty((0, size), dtype=np.float64), np.empty((0, size, size), dtype=np.float64)
        batch = getattr(self.solver_type, "batch_fisher_terms", None)
        if out is None and batch is not None and (len(self.white_noise) or len(self.kernel)):
            out = self._batch_fisher_device(batch, vectors, y, quiet)
        if out is None:
            res = self._batch_loop(vectors, lambda: self.fisher_information(y, quiet=quiet))
            if y is None:
                return np.stack(res)
            out = np.stack([r[0] for r in res]), np.stack([r[1] for r in res])
        return out if y is not None else out[1]

    def _batch_fisher_device(self, batch, vectors, y, quiet):
        """The batched dense path of :func:`batch_fisher_information`: ``(grad, F)``, or ``None`` when the kernel has
        no valid device program or more than ``_MAX_GRAD_PARAMS`` parameters."""
        members = self._batch_predict_members(vectors, y)  # GP._residual, the single call's residual
        if members is None or members[2].shape[1] > _MAX_GRAD_PARAMS:
            return None
        spec, full, kpar, sigma, resid, fact_err, mean_err = members
        nb, n, size = len(vectors), len(self._x), len(self)
        layout = n_mean, n_wn, n_k = self._grad_layout()
        mask = self.kernel.unfrozen_mask
        # each member's white-noise vectors and mean gradient, the device's inputs, with the single call's operations;
        # a member's first failure here is kept for the loop over the members below
        wn_full = slice(self.mean.full_size, self.mean.full_size + self.white_noise.full_size)
        noise, dmu, late_err = [None] * nb, [None] * nb, [None] * nb
        v = np.zeros((nb, n_wn, n), dtype=np.float64)
        dmu_in = np.zeros((nb, n_mean, n), dtype=np.float64)
        for b in range(nb):
            try:
                if n_wn:
                    noise[b] = self._swap_eval(self.white_noise, full[b, wn_full], self._white_noise_terms)
                    v[b] = np.exp(noise[b][0])[None, :] * noise[b][1]
                dmu[b] = self._member_gradients(layout, full[b])[0]
                if n_mean:
                    d = np.array(dmu[b].T, dtype=np.float64, order="F")
                    _check_finite(d)  # BasicSolver.apply_inverse's check, which the single call's solve meets
                    dmu_in[b] = d.T
            except Exception as exc:
                late_err[b] = exc
        gterms, rows, rdiag, kdmu, info = batch(spec, kpar, self._x, sigma, resid, mask.astype(np.uint32), v, dmu_in)
        grad = np.zeros((nb, size), dtype=np.float64)
        F = np.zeros((nb, size, size), dtype=np.float64)
        for b in range(nb):  # the loop's order: factorisation (white noise included), residual, white noise, mean
            if self._member_failed(spec, kpar, b, info, fact_err, mean_err, quiet, True):
                continue
            if late_err[b] is not None:
                if quiet and isinstance(late_err[b], ValueError):
                    continue
                raise late_err[b]
            self._fisher_matrix(F[b], layout, dmu[b], kdmu[b].T, rows[b][:, mask], rdiag[b], v[b])
            if y is not None:
                alpha, g, diag = gterms
                self._grad_row(grad[b], layout, dmu[b], alpha[b], lambda: noise[b], diag[b], g[b], mask, 0.5)
        return grad, F

    def _fisher_rows_host(self, v, n_k):
        """``(rows, rdiag)`` as ``BasicSolver.fisher_terms`` returns them (active kernel columns only), on the host:
        ``B = K^-1 dK K^-1`` for each active kernel parameter, then each white-noise vector (``dK = diag(v_k)``), with
        ``K^-1 = solver.apply_inverse(eye(N))`` and ``dK_p`` from ``kernel.get_gradient``."""
        n = len(self._x)
        kinv = np.asarray(self.solver.apply_inverse(np.eye(n), in_place=True), dtype=np.float64).reshape(n, n)
        dK = self.kernel.get_gradient(self._x) if n_k else np.zeros((n, n, 0))
        planes = [kinv.dot(dK[:, :, p]).dot(kinv) for p in range(n_k)]
        planes += [kinv.T.dot(vk[:, None] * kinv) for vk in v]
        rows = np.array([np.einsum("ij,ijq->q", B, dK) for B in planes]).reshape(len(planes), n_k)
        rdiag = np.array([np.diag(B) for B in planes]).reshape(len(planes), n)
        return rows, rdiag

    # -- leave-one-out cross-validation (Rasmussen & Williams, GPML §5.4.2, eqs. 5.10-5.13) ---------------------------
    def loo_predict(self, y):
        """The leave-one-out predictive of each observation at the computed coordinates: ``(mu, var)``, each of shape
        ``(N,)``, the mean and variance of ``y_i`` given all the other points, from one factorisation:
        ``mu_i = y_i - alpha_i / d_i`` and ``var_i = 1 / d_i`` with ``alpha = K^-1 (y - mean)`` and ``d = diag(K^-1)``.
        ``var`` includes the white noise and ``yerr``.  ``(y - mu) / sqrt(var)`` are the standardised LOO residuals.

        The HODLR solvers give the LOO quantities of their HODLR matrix ``K~``, not of the dense ``K``."""
        self.recompute(quiet=False)
        y = np.asarray(self._check_dimensions(y), dtype=np.float64)
        alpha, d = self._loo_terms(self._residual_of(y), None)
        return y - alpha / d, 1.0 / d

    def loo_log_likelihood(self, y, quiet=False):
        """The leave-one-out log predictive probability ``sum_i log p(y_i | y_-i)`` (GPML eq. 5.11), a model-selection
        score that is less sensitive to a mis-specified model than :func:`log_likelihood`:
        ``sum_i [-1/2 log(2 pi) + 1/2 log d_i - alpha_i^2 / (2 d_i)]`` with ``alpha`` and ``d`` as in
        :func:`loo_predict`.  Semantics follow :func:`log_likelihood`: ``-inf`` on a factorisation or mean-function
        failure when ``quiet``, and for a non-finite result (including a ``d_i`` that is not finite and positive, which
        a loose-tolerance HODLR matrix can give).

        The HODLR solvers give the LOO quantities of their HODLR matrix ``K~``, not of the dense ``K``."""
        if not self.recompute(quiet=quiet):
            return -np.inf
        try:
            r = self._residual_of(y)
        except ValueError as exc:
            if quiet and "mean function" in str(exc):
                return -np.inf
            raise
        alpha, d = self._loo_terms(r, None)
        return self._loo_value(alpha, d)

    def grad_loo_log_likelihood(self, y, quiet=False, return_value=False):
        """Gradient of :func:`loo_log_likelihood` w.r.t. the active parameter vector, in :func:`grad_log_likelihood`'s
        layout (mean, white noise, kernel; frozen parameters left out), from one factorisation (GPML eqs. 5.12-5.13):
        with ``beta = K^-1 (alpha / d)``, ``c = (1 + alpha**2 / d) / (2 d)`` and
        ``A = 1/2 (beta alpha^T + alpha beta^T) - K^-1 diag(c) K^-1``, the kernel part is ``sum_ij A_ij dK_ij/dtheta``,
        the white-noise part ``sum_i A_ii exp(wn_i) dwn_i/dtheta`` and the mean part ``dmu/dtheta . beta``.  Use it as
        ``scipy.optimize.minimize(..., jac=True)``'s objective with ``return_value``, which returns
        ``(loo_log_likelihood, grad)`` from the same pass, the value bit for bit what :func:`loo_log_likelihood` returns.

        A ``d_i`` that is not finite and positive raises ``ValueError`` naming the point.  With ``quiet`` any failure
        that :func:`grad_log_likelihood` absorbs gives a zero gradient (and ``-inf`` for the value).

        Solvers with a ``loo_terms`` hook (``BasicSolver``, ``HODLRSolver``) run on the device and never form K^-1 on
        the host; any other solver forms ``K^-1`` with ``apply_inverse`` on the host.  The HODLR solvers give the LOO
        quantities of their HODLR matrix ``K~``, not of the dense ``K``."""
        nothing = np.zeros(len(self), dtype=np.float64)
        fail = (-np.inf, nothing) if return_value else nothing
        if not self.recompute(quiet=quiet):
            return fail
        layout = self._grad_layout()
        mask = self.kernel.unfrozen_mask
        try:
            r = self._residual_of(y)
            alpha, d, beta, gk, diagA = self._loo_terms(r, mask.astype(np.uint32))
            dmu = self._call_mean_gradient(self._x) if layout[0] else None
        except ValueError:
            if quiet:
                return fail
            raise
        grad = self._grad_row(np.empty(len(self)), layout, dmu, beta, self._white_noise_terms, diagA, gk, mask, 1.0)
        return (self._loo_value(alpha, d), grad) if return_value else grad

    @staticmethod
    def _loo_value(alpha, d):
        """``sum_i [-1/2 log(2 pi) + 1/2 log d_i - alpha_i^2 / (2 d_i)]``; ``-inf`` unless every ``d_i`` is finite and
        positive and the sum is finite."""
        if not np.all(np.isfinite(d) & (d > 0)):
            return -np.inf
        v = float(np.sum(-0.5 * np.log(2 * np.pi) + 0.5 * np.log(d) - alpha ** 2 / (2 * d)))
        return v if np.isfinite(v) else -np.inf

    def _loo_terms(self, r, which):
        """``(alpha, d)``, or with ``which`` (0/1 over all kernel parameters) ``(alpha, d, beta, g, diagA)``, as
        ``BasicSolver.loo_terms`` returns them: from the solver's ``loo_terms`` hook, or on the host from
        ``K^-1 = solver.apply_inverse(eye(N))`` and ``KernelInterface.gradient_contract`` (``TrivialSolver``, plug-in
        solvers and a dense solver restored from a pickle)."""
        hook = getattr(self.solver, "loo_terms", None)
        if hook is not None:
            terms = hook(r, which)
            if terms is not None:
                return terms
        n = len(r)
        kinv = np.asarray(self.solver.apply_inverse(np.eye(n), in_place=True), dtype=np.float64).reshape(n, n)
        alpha = kinv.dot(r)
        d = np.diag(kinv).copy()
        if which is None:
            return alpha, d
        bad = np.flatnonzero(~(np.isfinite(d) & (d > 0)))
        if bad.size:
            raise ValueError("leave-one-out: diag(K^-1) at point {0} is {1:g}, not a finite positive number".format(
                bad[0], d[bad[0]]))
        q = alpha / d
        beta = kinv.dot(q)
        c = (1.0 + alpha * q) / (2.0 * d)
        A = 0.5 * (np.outer(beta, alpha) + np.outer(alpha, beta)) - kinv.dot(c[:, None] * kinv)
        g = np.zeros(len(which), dtype=np.float64)
        if len(which):
            g = self.kernel.kernel.gradient_contract(which, self._x, A)
        return alpha, d, beta, g, np.diag(A).copy()

    def batch_loo_predict(self, vectors, y):
        """:func:`loo_predict` at many parameter vectors: ``(mu, var)``, each ``(B, N)``, row ``b`` bit for bit what
        ``gp.set_parameter_vector(vectors[b]); gp.loo_predict(y)`` returns on the computed ``x`` and ``yerr``: the
        standardised LOO residuals ``(y - mu) / sqrt(var)`` of every sample of a posterior chain in one call, for
        calibration and outlier checks.  See :func:`batch_grad_loo_log_likelihood` for the errors, the GP's state and
        which solvers run batched.

        :param vectors: ``(B, len(gp))`` active-parameter vectors, as :func:`set_parameter_vector` takes them
        """
        return self._batch_loo("predict", vectors, y, False, False)

    def batch_loo_log_likelihood(self, vectors, y, quiet=False):
        """:func:`loo_log_likelihood` at many parameter vectors: entry ``b`` of the ``(B,)`` result is bit for bit what
        ``gp.set_parameter_vector(vectors[b]); gp.loo_log_likelihood(y, quiet=quiet)`` returns on the computed ``x``
        and ``yerr``.  See :func:`batch_grad_loo_log_likelihood` for the errors, the GP's state and which solvers run
        batched.

        :param vectors: ``(B, len(gp))`` active-parameter vectors, as :func:`set_parameter_vector` takes them
        """
        return self._batch_loo("value", vectors, y, quiet, False)

    def batch_grad_loo_log_likelihood(self, vectors, y, quiet=False, return_value=False):
        """:func:`grad_loo_log_likelihood` at many parameter vectors: row ``b`` of the ``(B, len(gp))`` result is bit
        for bit what ``gp.set_parameter_vector(vectors[b]); gp.grad_loo_log_likelihood(y, quiet=quiet,
        return_value=return_value)`` returns on the computed ``x`` and ``yerr``; with ``return_value`` the result is
        ``(value, grad)``, ``value`` of shape ``(B,)``.  The values and gradients of every start of a multi-start LOO
        fit (an objective more multimodal than the marginal likelihood) in one call.

        With ``quiet`` a failing member gets the loop's ``-inf`` and zero gradient and the others are unaffected;
        otherwise the exception that loop raises first is raised, with its type and message (white noise or
        factorisation, then the residual, then a ``d_i`` that is not finite and positive, then the mean gradient),
        with one difference: the checks that do not depend on the member (the shape of ``vectors``, ``y``'s length)
        come first.  The GP is left as it was: parameter vector, factorisation, cached solve and dirty flags.

        Solvers with a ``batch_loo_terms`` hook (``BasicSolver``) factorise all members, form their ``K^-1`` and
        contract the kernel gradients in one batched pass on the device.  Any other solver (``HODLRSolver``,
        ``TrivialSolver``, ``ShardedHODLRSolver``, plug-ins) takes that loop, and so do a kernel without a valid device
        program and, for the gradient, one with more than 64 parameters (the device contraction's limit: every
        member's gradient then fails as it does in the loop).

        :param vectors: ``(B, len(gp))`` active-parameter vectors, as :func:`set_parameter_vector` takes them
        """
        return self._batch_loo("grad", vectors, y, quiet, return_value)

    def _batch_loo(self, kind, vectors, y, quiet, return_value):
        """The three ``batch_*loo*`` methods: ``kind`` is ``"predict"``, ``"value"`` or ``"grad"``."""
        vectors = self._batch_vectors(vectors)
        self._check_dimensions(y)
        nb, n = len(vectors), len(self._x)
        if nb == 0:
            if kind == "predict":
                return np.empty((0, n), dtype=np.float64), np.empty((0, n), dtype=np.float64)
            value, grad = np.empty(0, dtype=np.float64), np.empty((0, len(self)), dtype=np.float64)
            return value if kind == "value" else ((value, grad) if return_value else grad)
        batch = getattr(self.solver_type, "batch_loo_terms", None)
        if batch is not None:
            out = self._batch_loo_device(batch, kind, vectors, y, quiet, return_value)
            if out is not None:
                return out
        if kind == "predict":
            res = self._batch_loop(vectors, lambda: self.loo_predict(y))
            return np.stack([r[0] for r in res]), np.stack([r[1] for r in res])
        if kind == "value":
            return np.array(self._batch_loop(vectors, lambda: self.loo_log_likelihood(y, quiet=quiet)),
                            dtype=np.float64)
        res = self._batch_loop(vectors, lambda: self.grad_loo_log_likelihood(y, quiet=quiet, return_value=True))
        value, grad = np.array([r[0] for r in res], dtype=np.float64), np.stack([r[1] for r in res])
        return (value, grad) if return_value else grad

    def _batch_loo_device(self, batch, kind, vectors, y, quiet, return_value):
        """The batched dense path of :func:`_batch_loo`; ``None`` when the kernel has no valid device program or, for
        the gradient, more than ``_MAX_GRAD_PARAMS`` parameters."""
        members = self._batch_members(vectors, y, self._residual_of,
                                      lambda y, c: y if c == 0.0 else y - c)  # the operations of GP._residual_of
        if members is None or (kind == "grad" and members[2].shape[1] > _MAX_GRAD_PARAMS):
            return None
        spec, full, kpar, sigma, resid, fact_err, mean_err = members
        nb = len(vectors)
        if kind == "predict":
            alpha, d, info = batch(spec, kpar, self._x, sigma, resid)
            self._raise_member_error(spec, kpar, info, fact_err, mean_err)
            y = np.asarray(self._check_dimensions(y), dtype=np.float64)
            return y - alpha / d, 1.0 / d
        grad = kind == "grad"
        if grad:
            mask = self.kernel.unfrozen_mask
            alpha, d, beta, g, diag, info = batch(spec, kpar, self._x, sigma, resid, mask.astype(np.uint32))
        else:
            alpha, d, info = batch(spec, kpar, self._x, sigma, resid)
        # GP.loo_log_likelihood / GP.grad_loo_log_likelihood member by member, with their operations
        layout = self._grad_layout()
        value = np.full(nb, -np.inf)
        out = np.zeros((nb, len(self)), dtype=np.float64)
        for b in range(nb):  # the loop's order: factorisation (white noise included), residual, d, mean gradient
            if self._member_failed(spec, kpar, b, info, fact_err, mean_err, quiet, grad):
                continue
            if not grad:
                value[b] = self._loo_value(alpha[b], d[b])
                continue
            bad = np.flatnonzero(~(np.isfinite(d[b]) & (d[b] > 0)))
            try:
                if bad.size:  # the single call's check, raised there by the solver
                    raise ValueError("leave-one-out: diag(K^-1) at point {0} is {1:g}, not a finite positive "
                                     "number".format(bad[0], d[b, bad[0]]))
                dmu, noise = self._member_gradients(layout, full[b])
            except ValueError:
                if quiet:
                    continue
                raise
            self._grad_row(out[b], layout, dmu, beta[b], noise, diag[b], g[b], mask, 1.0)
            value[b] = self._loo_value(alpha[b], d[b])
        if not grad:
            return value
        return (value, out) if return_value else out

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
        vectors = self._batch_vectors(vectors)
        self._check_dimensions(y)
        out = None
        if len(vectors) == 0:
            out = np.empty(0, dtype=np.float64), np.empty((0, len(self)), dtype=np.float64)
        batch = getattr(self.solver_type, "batch_grad_terms", None)
        if out is None and batch is not None and (len(self.white_noise) or len(self.kernel)):
            out = self._batch_grad_device(batch, vectors, y, quiet, return_log_likelihood)
        if out is None:
            res = self._batch_loop(vectors, lambda: (self.log_likelihood(y, quiet=quiet) if return_log_likelihood
                                                     else np.nan, self.grad_log_likelihood(y, quiet=quiet)))
            out = np.array([r[0] for r in res], dtype=np.float64), np.stack([r[1] for r in res])
        return out if return_log_likelihood else out[1]

    def _batch_grad_device(self, batch, vectors, y, quiet, return_ll):
        """The batched dense path of :func:`batch_grad_log_likelihood`: ``(ll, grad)``, or ``None`` when the kernel
        has no valid device program or more than ``_MAX_GRAD_PARAMS`` parameters."""
        # one residual serves both terms: GP._residual (the gradient's) and GP._residual_of (the value's) round alike
        members = self._batch_predict_members(vectors, y)
        if members is None or members[2].shape[1] > _MAX_GRAD_PARAMS:
            return None
        spec, full, kpar, sigma, resid, fact_err, mean_err = members
        nb = len(vectors)
        mask = self.kernel.unfrozen_mask
        log_det, quad, alpha, g, diag, info = batch(spec, kpar, self._x, sigma, resid, mask.astype(np.uint32))
        ll = self._batch_ll(log_det, quad)
        # GP.grad_log_likelihood member by member, with its operations
        layout = self._grad_layout()
        grad = np.zeros((nb, len(self)), dtype=np.float64)
        for b in range(nb):  # the loop's order: factorisation (white noise included), residual, mean gradient
            # (with the value, the loop's log_likelihood comes first and lets a residual ValueError through)
            if self._member_failed(spec, kpar, b, info, fact_err, mean_err, quiet, not return_ll):
                ll[b] = -np.inf
                continue
            try:
                dmu, noise = self._member_gradients(layout, full[b])
            except ValueError:
                if quiet:
                    continue
                raise
            self._grad_row(grad[b], layout, dmu, alpha[b], noise, diag[b], g[b], mask, 0.5)
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
            return self._predict_mean(alpha, xs, kernel)
        return self._predict_spread(alpha, xs, return_var, kernel)

    def _predict_mean(self, alpha, xs, kernel):
        """K(x*, x) alpha + mean(x*), K(x*, x) alpha evaluated matrix-free on the device (csrc/kmat_ops.cu); the
        reference forms the (n*, N) matrix on the host (gp.py:524-528), which stops being possible long before
        N = 2^18."""
        return kernel.matvec(xs, self._x, alpha) + self._call_mean(xs)

    def _predict_spread(self, alpha, xs, return_var, kernel):
        """``(mu, var)`` or ``(mu, cov)`` of :func:`predict`."""
        # variance / covariance from the stored factorisation on the device (BasicSolver, HODLRSolver): K(x*, x) and
        # K^-1 K(x, x*) stay there, streamed in column chunks.  Solvers without `predictive`, or that return None (a
        # pickled dense factor, a sharded tree), take the reference's host route below.
        predictive = getattr(self.solver, "predictive", None)
        out = predictive(kernel, xs, "var" if return_var else "cov") if predictive is not None else None
        if out is not None:
            return self._predict_mean(alpha, xs, kernel), out
        return self._predict_host(alpha, xs, return_var, kernel)

    def _predict_host(self, alpha, xs, return_var, kernel):
        """The reference's route (gp.py:534-545): K(x*, x) on the host, ``solver.apply_inverse`` on its transpose."""
        Kxs = kernel.get_value(xs, self._x)
        mu = np.dot(Kxs, alpha) + self._call_mean(xs)

        KinvKxs = self.solver.apply_inverse(Kxs.T)
        if return_var:
            return mu, self._host_var(Kxs, KinvKxs, xs, kernel)
        cov = kernel.get_value(xs)
        cov -= np.dot(Kxs, KinvKxs)
        return mu, cov

    @staticmethod
    def _host_var(Kxs, KinvKxs, xs, kernel):
        var = kernel.get_value(xs, diag=True)
        var -= np.sum(Kxs.T * KinvKxs, axis=0)
        return var

    def grad_predict(self, y, t, return_var=False, cache=True, kernel=None):
        """The predictive mean (and variance) at ``t`` with their gradients with respect to the test points:
        ``(mu, dmu)``, or ``(mu, var, dmu, dvar)`` with ``return_var``.  ``mu`` and ``var`` (``(ns,)``) are bit for bit
        what :func:`predict` returns with ``return_cov=False`` / ``return_var=True`` and the same ``cache`` and
        ``kernel``; ``dmu[i, q] = d mu_i / d t_iq`` and ``dvar[i, q] = d var_i / d t_iq`` (``(ns, ndim)``, also for a
        1-D ``t``).  Each output depends on its own test point only, so this is the whole Jacobian: what an optimiser
        of an acquisition function (``mu + kappa * sqrt(var)``, expected improvement) needs per step.

        With ``B = K(x, t)`` and ``W = K^-1 B``: ``dmu_i = sum_j d1 k(t_i, x_j) alpha_j`` and ``dvar_i = d k(t_i, t_i)
        / d t_i - 2 sum_j d1 k(t_i, x_j) W_ji``, the true derivatives for every metric (:func:`Kernel.get_x1_gradient`
        keeps the reference's values, which differ for a general metric).  The contractions run on the device without
        the ``(ns, N, ndim)`` gradient tensor; ``BasicSolver`` and ``HODLRSolver`` stream ``var`` and ``dvar`` through
        the stored factorisation (``predictive_grad``), ``ShardedHODLRSolver`` likewise with each rank contracting its
        own rows (collective), and every other solver (``TrivialSolver``, a pickled dense solver, plug-ins without a
        ``predictive_grad`` hook) contracts the ``solver.apply_inverse(B)`` of :func:`predict`'s host route.

        A ``ConstantModel`` mean adds nothing to ``dmu``; any other mean model raises ``NotImplementedError`` (the
        modeling protocol has no input gradient).  Inputs of more than 8 dimensions raise ``ValueError``.
        """
        _check_grad_predict_mean(self.mean)
        self._require_computed()
        xs = self.parse_samples(t)
        _check_grad_predict_dim(xs)
        self.recompute()
        alpha = self._compute_alpha(y, cache)
        if kernel is None:
            kernel = self.kernel
        mu = self._predict_mean(alpha, xs, kernel)
        dmu = kernel.kernel.x1_gradient_matvec(xs, self._x, alpha)
        if not return_var:
            return mu, dmu
        hook = getattr(self.solver, "predictive_grad", None)
        out = hook(kernel, xs) if hook is not None else None
        if out is None:
            Kxs = kernel.get_value(xs, self._x)
            KinvKxs = self.solver.apply_inverse(Kxs.T)
            out = (self._host_var(Kxs, KinvKxs, xs, kernel),
                   kernel.kernel.x1_gradient_matvec(xs, self._x, KinvKxs, scale=-2.0, add_prior=True))
        var, dvar = out
        return mu, var, dmu, dvar

    def batch_grad_predict(self, vectors, y, t, return_var=False, kernel=None):
        """:func:`grad_predict` at many parameter vectors: ``(mu, dmu)``, or ``(mu, var, dmu, dvar)`` with
        ``return_var``; ``mu`` and ``var`` are ``(B, ns)``, ``dmu`` and ``dvar`` ``(B, ns, ndim)`` (also for a 1-D
        ``t``).  Entry ``b`` is bit for bit what ``gp.set_parameter_vector(vectors[b]); gp.grad_predict(y, t,
        return_var=...)`` returns on the computed ``x`` and ``yerr``: an acquisition function averaged over a sampler's
        chain (the integrated acquisition of Snoek, Larochelle and Adams, 2012) and its gradient in one call.  The GP
        is left as it was: parameter vector, factorisation, cached solve and dirty flags.

        The checks that do not depend on the member come first, with :func:`grad_predict`'s and :func:`batch_predict`'s
        exceptions: a mean model other than a ``ConstantModel`` (``NotImplementedError``), a model that has not been
        computed, the shape of ``vectors``, ``y``'s length, ``t``'s dimension and more than 8 input dimensions.  Then
        a failing member raises the exception the loop would raise first, with its type and message (white noise,
        factorisation, residual).  With no members or no test points nothing is computed and the empty results are
        returned.

        Solvers with a ``batch_predict_grad`` hook (``BasicSolver``) factorise all members and compute their means,
        variances and gradients in one batched pass on the device; any other solver (``HODLRSolver``,
        ``ShardedHODLRSolver``, ``TrivialSolver``, plug-ins), an explicit ``kernel`` and a kernel without a valid
        device program take that loop.

        :param vectors: ``(B, len(gp))`` active-parameter vectors, as :func:`set_parameter_vector` takes them
        """
        _check_grad_predict_mean(self.mean)
        vectors = self._batch_vectors(vectors)
        self._check_dimensions(y)
        xs = self.parse_samples(t)
        _check_grad_predict_dim(xs)
        nb, ns, nd = len(vectors), len(xs), xs.shape[1]
        if nb == 0 or ns == 0:
            mu, dmu = np.empty((nb, ns), dtype=np.float64), np.empty((nb, ns, nd), dtype=np.float64)
            if not return_var:
                return mu, dmu
            return mu, np.empty((nb, ns), dtype=np.float64), dmu, np.empty((nb, ns, nd), dtype=np.float64)
        batch = getattr(self.solver_type, "batch_predict_grad", None)
        if batch is not None and kernel is None:
            out = self._batch_grad_predict_device(batch, vectors, y, xs, return_var)
            if out is not None:
                return out
        res = self._batch_loop(vectors, lambda: self.grad_predict(y, t, return_var=return_var, kernel=kernel))
        return tuple(np.stack([r[k] for r in res]) for k in range(len(res[0])))

    def _batch_grad_predict_device(self, batch, vectors, y, xs, return_var):
        """The batched dense path of :func:`batch_grad_predict`; ``None`` when the kernel has no valid device
        program."""
        members = self._batch_predict_members(vectors, y)
        if members is None:
            return None
        spec, full, kpar, sigma, resid, fact_err, mean_err = members
        mean_xs, xs_err = self._batch_mean_at(full, xs)
        mu, var, dmu, dvar, info = batch(spec, kpar, self._x, sigma, resid, xs, return_var)
        self._raise_member_error(spec, kpar, info, fact_err, mean_err, xs_err)  # residual, mean at x*
        mu += mean_xs  # a constant mean adds nothing to dmu
        return (mu, var, dmu, dvar) if return_var else (mu, dmu)

    def sample_conditional(self, y, t, size=1, *, rng=None, jitter=None):
        """Draws from the conditional predictive distribution at ``t``: shape ``(ns,)`` when ``size == 1``, else
        ``(size, ns)``.

        With ``rng=None`` this is the reference's route: ``predict(y, t)`` and ``numpy.random.multivariate_normal``
        (an SVD of the covariance on the host, drawing from numpy's global generator).

        With ``rng`` (a ``numpy.random.Generator`` or ``RandomState``) the draws are ``mu + z @ L.T``, where ``z =
        rng.standard_normal((size, ns))`` is drawn exactly once, after the argument checks and before any device call,
        ``(mu, C)`` is what ``predict(y, t, return_cov=True)`` returns and ``L`` is the lower Cholesky factor of
        ``sym(C) + jitter * I`` computed on the device, ``sym(C)`` mirroring the lower triangle of ``C`` (the HODLR
        covariance is symmetric only to ``tol``).  ``jitter`` defaults to ``TINY``.  ``BasicSolver`` and
        ``HODLRSolver`` build ``C`` on the device and never copy it to the host (``sample_predictive``); other
        solvers sample from ``predict``'s covariance.  On ``ShardedHODLRSolver`` every rank returns the same draws
        provided ``rng`` is seeded identically on every rank, as ``y`` and ``t`` are replicated.

        If that matrix is not positive definite (a negative predictive variance, a NaN) the call raises
        ``numpy.linalg.LinAlgError`` naming the failed leading minor, where the host route warns and draws anyway; the
        GP stays as it was.
        """
        jitter = _sampling_jitter(rng, jitter)
        if rng is None:
            mu, cov = self.predict(y, t)
            return multivariate_gaussian_samples(cov, size, mean=mu)
        size = _check_size(size)
        self._require_computed()
        self._check_dimensions(y)
        xs = self.parse_samples(t)
        z = rng.standard_normal((size, len(xs)))
        if size == 0:
            return np.empty((0, len(xs)), dtype=np.float64)
        self.recompute()
        alpha = self._compute_alpha(y, True)
        draws = None
        fused = getattr(self.solver, "sample_predictive", None)
        if fused is not None:
            draws = fused(self.kernel, xs, self._predict_mean(alpha, xs, self.kernel), z, jitter)
        if draws is None:
            mu, cov = self._predict_spread(alpha, xs, False, self.kernel)
            draws = device_gaussian_samples(cov, z, mu, jitter)
        return draws[0] if size == 1 else draws

    def batch_sample_conditional(self, vectors, y, t, size=1, *, rng=None, jitter=None):
        """:func:`sample_conditional` at many parameter vectors: ``(B, ns)`` when ``size == 1``, else ``(B, size,
        ns)``, entry ``b`` being bit for bit what ``gp.set_parameter_vector(vectors[b]); gp.sample_conditional(y, t,
        size, rng=rng, jitter=jitter)`` returns, run over ``b`` in order on the computed ``x`` and ``yerr``: posterior
        predictive draws for each sample of a chain in one call.  The GP is left as it was: parameter vector,
        factorisation, cached solve and dirty flags.

        With ``rng`` (a ``numpy.random.Generator`` or ``RandomState``) the normals are drawn on the host, one
        ``rng.standard_normal((size, ns))`` per member in member order, all of them after the argument checks and
        before any device call.  When no member fails the generator ends where that loop leaves it; when one fails it
        has still advanced by all ``B`` members' normals.  ``rng=None`` runs that loop itself (the reference's host
        route, numpy's global generator).

        The argument checks (``rng``, ``jitter``, ``size``, a computed model, the shape of ``vectors``, ``y``'s length,
        ``t``'s dimension) come first and raise what :func:`sample_conditional` (or, for ``vectors``,
        :func:`batch_predict`) raises.  Then a failing member raises the exception the loop would raise first, with its
        type and message: white noise, factorisation, residual, mean at ``t``, and a predictive covariance that is not
        positive definite.  With no members, ``size == 0`` or no test points nothing is computed and the empty result
        is returned, the generator advanced as the loop would advance it; with no test points the loop would still
        factorise every member, which is skipped here as in :func:`batch_predict`.

        Solvers with a ``batch_sample`` hook (``BasicSolver``) factorise, predict and draw for all members in one
        batched pass on the device; any other solver (``HODLRSolver``, ``ShardedHODLRSolver``, ``TrivialSolver``,
        plug-ins) and a kernel without a valid device program take that loop.

        :param vectors: ``(B, len(gp))`` active-parameter vectors, as :func:`set_parameter_vector` takes them
        """
        jitter = _sampling_jitter(rng, jitter)
        size = _check_size(size)
        vectors = self._batch_vectors(vectors)
        self._check_dimensions(y)
        xs = self.parse_samples(t)
        nb, ns = len(vectors), len(xs)
        shape = (nb, ns) if size == 1 else (nb, size, ns)
        if nb == 0:
            return np.empty(shape, dtype=np.float64)
        if rng is not None and (size == 0 or ns == 0):
            for _ in range(nb):
                rng.standard_normal((size, ns))
            return np.empty(shape, dtype=np.float64)
        batch = getattr(self.solver_type, "batch_sample", None)
        if batch is not None and rng is not None:
            out = self._batch_sample_device(batch, vectors, y, xs, size, rng, jitter)
            if out is not None:
                return out
        return np.stack(self._batch_loop(vectors, lambda: self.sample_conditional(y, t, size, rng=rng, jitter=jitter)))

    def _batch_sample_device(self, batch, vectors, y, xs, size, rng, jitter):
        """The batched dense path of :func:`batch_sample_conditional`; ``None`` when the kernel has no valid device
        program (nothing has been drawn from ``rng`` then)."""
        members = self._batch_predict_members(vectors, y)
        if members is None:
            return None
        spec, full, kpar, sigma, resid, fact_err, mean_err = members
        nb, ns = len(vectors), len(xs)
        z = np.empty((nb, size, ns), dtype=np.float64)
        for b in range(nb):
            z[b] = rng.standard_normal((size, ns))
        mean_xs, xs_err = self._batch_mean_at(full, xs)
        draws, info, draw_info = batch(spec, kpar, self._x, sigma, resid, xs, mean_xs, z, jitter)
        cov_err = [LinAlgError("%d-th leading minor of the array is not positive definite (a larger jitter adds more "
                               "to the diagonal)" % d) if d != 0 else None for d in draw_info]
        self._raise_member_error(spec, kpar, info, fact_err, mean_err, xs_err, cov_err)  # residual, mean at x*, cov
        return draws[:, 0] if size == 1 else draws

    def sample(self, t=None, size=1, *, rng=None):
        """Draw from the prior, at ``t`` or (``t is None``) at the computed coordinates via the Cholesky factor.

        With ``rng=None`` this is the reference's route (numpy's global generator; at ``t``, an SVD of
        ``K(t, t) + TINY`` on the host).  With ``rng`` (a ``numpy.random.Generator`` or ``RandomState``) the normals are
        ``rng.standard_normal((size, n))``, drawn once after the argument checks: at ``t`` the draws are those of
        :func:`sample_conditional` with ``mu = mean(t)``, ``C = K(t, t)`` and ``jitter = TINY``; with ``t=None`` they
        are ``solver.sample_prior(z) + mean(x)`` on a solver with that hook (``HODLRSolver``), else
        ``solver.apply_sqrt(z) + mean(x)``.

        ``HODLRSolver`` draws through the symmetric factor ``K~ = W W^T`` of its HODLR matrix ``K~`` (built on the
        device on first use after a ``compute``): the draws ``W z + mean`` are distributed as ``N(mean, K~)``, but they
        are not the dense solver's draws for the same ``z``, whose square root is the Cholesky factor.  A ``K~`` that
        is not positive definite raises ``numpy.linalg.LinAlgError`` and leaves the GP as it was.  With ``rng=None``
        the route stays the reference's, ``apply_sqrt``, which ``HODLRSolver`` does not implement."""
        if rng is None:
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
        _check_rng(rng)
        size = _check_size(size)
        if t is None:
            self._require_computed()
            z = rng.standard_normal((size, self._x.shape[0]))
            self.recompute()
            hook = getattr(self.solver, "sample_prior", None)
            draws = hook(z) if hook is not None else None
            if draws is None:
                draws = self.solver.apply_sqrt(z)
            draws += self._call_mean(self._x)
        else:
            x = self.parse_samples(t)
            z = rng.standard_normal((size, len(x)))
            if size == 0:
                return np.empty((0, len(x)), dtype=np.float64)
            draws = device_gaussian_samples(self.get_matrix(x), z, self._call_mean(x), TINY)
        return draws[0] if size == 1 else draws

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
