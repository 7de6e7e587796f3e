# -*- coding: utf-8 -*-
"""The device interpreter, the gradient contraction and the solvers at the size limits of a kernel program.

The rest of the suite sends small programs through the library (at most 6 differentiated hyper-parameters, 9 leaves, an
operand stack of 3, 5 input dimensions).  Here every device path that only larger programs reach runs against a plain
reference:

* 8 | 9 | 11 | 37 | 64 hyper-parameters: either side of the ``kmat_grad_contract_kernel<8>`` / ``<64>`` switch, the
  CO2 kernel of the hyper-parameter tutorial, a general metric on 8 axes and exactly the 64-parameter limit; 65 must be
  rejected by every gradient entry point, before anything is solved;
* an operand stack of 8 (``BGP_STACK``) on the 1-D fast interpreter and on the general one (value, hyper-parameter
  gradient, input gradient); 9 must be rejected;
* 16 leaves in 31 nodes (``BGP_MAX_LEAVES``), also through the 768-row HODLR leaves (``LF_MAX_LEAF``); 17 leaves do
  not fit in 32 nodes;
* input dimensions up to 100, past the point where a tile's coordinates fit in the shared memory of the kernel-matrix
  builds (from 56 / 59 dimensions) and of the matvec (from 29), on both sides of the ``ProfileND`` (ndim <= 3) /
  interpreter switch, and HODLR at its 32-dimension limit (33 must be rejected).

References: values and gradient tensors come from the CPU oracle, pinned bit for bit to the reference's compiled
kernel_interface on these same programs (``limits__`` digests in tests/golden/reference_kernel_interface.json);
contractions, log-determinants, solves, gradients of the log-likelihood and predictions come from that K in longdouble
(tests/hiprec.py).  Every measured error is recorded with ``record_property``."""
import numpy as np
import pytest

import hiprec
from golden.make_golden_kernel_interface import golden_digest

LD = hiprec.LD

# Bars, with the largest error measured on an H100 (all programs, n, solvers and rng modes of the test):
VALUE_RTOL, VALUE_ATOL = 1e-13, 1e-15  # values, elementwise; pow-based kernels included              (measured 2.3e-15)
GRAD_RTOL, GRAD_ATOL = 1e-12, 1e-14    # gradient tensors (measured 4.7e-14) and input gradients     (measured 4.3e-14)
MATVEC_TOL = 1e-14       # |Kv - ref| / (|K| |v|), elementwise                                        (measured 2.1e-16)
CONTRACT_TOL = 5e-15     # |g - g_ref| / sum |dK| |A|                                                 (measured 6.0e-17)
DOT_TOL = 1e-13          # batch: |r^T K^-1 r - ref| / |ref|                                           (measured 2.1e-15)
# solvers (cond(K) <= 1e4), measured dense | HODLR:
#   logdet   |logdet - ref| / max(1, |ref|)                                              1.5e-15 | 3.6e-15
#   solve    ||X - X_ref|| / ||X_ref||                                                   3.6e-14 | 1.3e-13
#   predict  mean / (|K(x*, x)| |alpha|) elementwise; var, cov / max |K(x*, x*)|         1.6e-15 | 6.5e-15
#   grad     grad_terms: alpha, diag as solve, g / sum |dK| |A|; GP.grad_log_likelihood:
#            each entry / the sum of the magnitudes of its terms                         6.8e-14 | 2.1e-13
DENSE_TOL = dict(logdet=5e-14, solve=2e-12, predict=1e-13, grad=5e-12)
HODLR_TOL = dict(logdet=2e-13, solve=1e-11, predict=2e-13, grad=2e-11)   # exact-K trees (tol 1e-15)

WIDE_NDIMS = [4, 8, 28, 29, 32, 33, 55, 56, 58, 59, 64, 100]
CONTRACT_N = [1, 31, 32, 33, 97, 300]   # GC_T = 32 tile edges


# ---- programs ------------------------------------------------------------------------------------------------------
def _general(nax, seed, scale):
    """A well-conditioned SPD metric matrix on nax axes."""
    a = np.random.default_rng(seed).normal(size=(nax, nax))
    return scale * (np.eye(nax) + 0.2 * a @ a.T / nax)


def _right_nested(leaves, ops):
    """leaves[0] op0 (leaves[1] op1 (... leaves[-1])): postfix l0 l1 ... lk op ... op, an operand stack of len(leaves)."""
    k = leaves[-1]
    for leaf, op in zip(leaves[-2::-1], ops[::-1]):
        k = leaf + k if op == "+" else leaf * k
    return k


def _co2_kernel(k1_amp=66.0 ** 2):
    from george_b200 import kernels as K
    k1 = k1_amp * K.ExpSquaredKernel(metric=67 ** 2)
    k2 = 2.4 ** 2 * K.ExpSquaredKernel(90 ** 2) * K.ExpSine2Kernel(gamma=2 / 1.3 ** 2, log_period=0.0)
    k3 = 0.66 ** 2 * K.RationalQuadraticKernel(log_alpha=np.log(0.78), metric=1.2 ** 2)
    k4 = 0.18 ** 2 * K.ExpSquaredKernel(1.6 ** 2)
    return k1 + k2 + k3 + k4


def _np64_kernel(matern_axes=4):
    """1 + 36 + 1 + 21 + 1 + 4 = 64 parameters (65 with the Matern on 5 axes), 8-D."""
    from george_b200 import kernels as K
    axes = list(range(8 - matern_axes, 8))
    return (1.0 * K.ExpSquaredKernel(_general(8, 3, 8.0), ndim=8)
            + 0.5 * K.ExpSquaredKernel(_general(6, 4, 6.0), ndim=8, axes=list(range(6)))
            + 0.3 * K.Matern32Kernel([1.0 + i for i in range(matern_axes)], ndim=8, axes=axes))


def _depth_1d_leaves():
    """Leaves the 1-D fast interpreter (BGP_FLAG_FAST1D) takes: scalar metrics, ExpSine2, Cosine, Constant."""
    from george_b200 import kernels as K
    return [K.ExpSquaredKernel(1.0), K.Matern32Kernel(2.0), K.Matern52Kernel(0.5), K.ExpKernel(1.5),
            K.RationalQuadraticKernel(log_alpha=0.2, metric=1.3), K.ExpSine2Kernel(gamma=1.2, log_period=0.3),
            K.CosineKernel(log_period=0.7), K.ConstantKernel(log_constant=-0.5), K.ExpSquaredKernel(3.0)]


def _depth_3d_kernel():
    from george_b200 import kernels as K
    leaves = [K.ExpSquaredKernel(_general(3, 5, 2.0), ndim=3), K.Matern32Kernel([0.5, 1.0, 2.0], ndim=3),
              K.ExpSine2Kernel(gamma=0.8, log_period=0.4, ndim=3, axes=1), K.Matern52Kernel(1.5, ndim=3, axes=[0, 2]),
              K.RationalQuadraticKernel(log_alpha=-0.3, metric=[1.0, 2.0], ndim=3, axes=[1, 2]),
              K.LocalGaussianKernel(location=0.1, log_width=0.5, ndim=3, axes=2),
              K.CosineKernel(log_period=0.9, ndim=3, axes=0), K.ExpKernel(2.0, ndim=3)]
    return _right_nested(leaves, ["*", "+", "*", "+", "*", "+", "*"])


def _sixteen_leaves(extra=False):
    """16 leaves of mixed types in 31 nodes, operand stack 4: the sum of four (a + b) * (c + d); `extra` adds a 17th."""
    from george_b200 import kernels as K
    L = [K.ExpSquaredKernel(1.5, ndim=3), K.ExpSquaredKernel([0.8, 1.5, 2.5], ndim=3),
         K.ExpSquaredKernel(_general(2, 6, 1.5), ndim=3, axes=[0, 2]), K.Matern32Kernel(2.0, ndim=3),
         K.Matern52Kernel(_general(3, 7, 3.0), ndim=3), K.ExpKernel(4.0, ndim=3, axes=2),
         K.RationalQuadraticKernel(log_alpha=0.4, metric=2.0, ndim=3), K.ExpSine2Kernel(gamma=0.6, log_period=0.8, ndim=3, axes=0),
         K.CosineKernel(log_period=1.1, ndim=3, axes=1), K.ConstantKernel(log_constant=-1.0, ndim=3),
         K.LocalGaussianKernel(location=-0.2, log_width=1.0, ndim=3, axes=0),
         K.ExpSquaredKernel(1.0, ndim=3, block=[(-3.0, 3.0)] * 3), K.Matern32Kernel([1.0, 3.0], ndim=3, axes=[0, 1]),
         K.ExpKernel(2.5, ndim=3, axes=[1, 2]), K.RationalQuadraticKernel(log_alpha=-0.2, metric=[1.5, 0.7, 2.0], ndim=3),
         K.Matern52Kernel(1.2, ndim=3, axes=1)]
    k = None
    for g in range(4):
        a, b, c, d = L[4 * g:4 * g + 4]
        term = (a + b) * (c + d)
        k = term if k is None else k + term
    return k + K.ConstantKernel(log_constant=0.0, ndim=3) if extra else k


def wide_kernel(nd):
    """A sum of leaves on disjoint blocks of at most 8 axes that cover every column (isotropic, axis-aligned and general
    metrics in turn), plus a leaf on axes [0, nd - 1]."""
    from george_b200 import kernels as K
    k = None
    for b, a0 in enumerate(range(0, nd, 8)):
        axes = list(range(a0, min(a0 + 8, nd)))
        na = len(axes)
        if b % 3 == 0:
            leaf = K.ExpSquaredKernel(2.0 * na, ndim=nd, axes=axes)
        elif b % 3 == 1:
            leaf = K.Matern32Kernel(list(2.0 * na * np.linspace(0.7, 1.3, na)), ndim=nd, axes=axes)
        else:
            leaf = K.Matern52Kernel(_general(na, 10 + b, 2.0 * na), ndim=nd, axes=axes)
        k = leaf if k is None else k + leaf
    return k + K.ExpKernel(3.0, ndim=nd, axes=[0, nd - 1])


def limit_programs():
    """(name, kernel) for every program the value / gradient tests run."""
    from george_b200 import kernels as K
    d1 = _depth_1d_leaves()
    out = [
        ("np8", 0.8 * K.ExpSquaredKernel(_general(3, 1, 2.0), ndim=3) + K.ConstantKernel(log_constant=-1.0, ndim=3)),
        ("np9", 0.8 * K.ExpSquaredKernel(_general(3, 1, 2.0), ndim=3)
         + K.ExpSine2Kernel(gamma=0.5, log_period=0.2, ndim=3, axes=1)),
        ("co2", _co2_kernel()),
        ("np37", 1.2 * K.ExpSquaredKernel(_general(8, 2, 8.0), ndim=8)),
        ("np64", _np64_kernel()),
        ("np65", _np64_kernel(5)),
        ("depth8_1d", _right_nested(d1[:8], ["+"] * 7)),
        ("depth8_3d", _depth_3d_kernel()),
        ("leaves16", _sixteen_leaves()),
    ]
    for d in (2, 3, 4):  # ProfileND (ndim <= 3) against the interpreter
        out.append(("iso_{0}d".format(d), 1.3 * K.ExpSquaredKernel(1.5, ndim=d)))
        out.append(("axis_{0}d".format(d), 0.7 * K.Matern32Kernel(list(np.linspace(0.8, 1.6, d)), ndim=d)))
    out += [("wide_{0}d".format(nd), wide_kernel(nd)) for nd in WIDE_NDIMS]
    return out


_PROGRAMS = dict(limit_programs())
NAMES = sorted(_PROGRAMS)
GRAD_NAMES = [n for n in NAMES if len(_PROGRAMS[n]) <= 64]
XGRAD_NAMES = [n for n in NAMES if _PROGRAMS[n].ndim <= 8]
CONTRACT_NAMES = ["np8", "np9", "co2", "np37", "np64", "depth8_1d", "depth8_3d", "leaves16"]


def _program(name):
    return _PROGRAMS[name]


def _err(a, ref, rtol, atol):
    """max |a - ref| / max(|ref|, atol / rtol): <= rtol exactly when |a - ref| <= max(rtol |ref|, atol) everywhere."""
    a, ref = np.asarray(a, dtype=LD), np.asarray(ref, dtype=LD)
    if a.size == 0:
        return 0.0
    return float(np.max(np.abs(a - ref) / np.maximum(np.abs(ref), LD(atol / rtol))))


def _rel(X, Xr):
    Xr = np.asarray(Xr, dtype=LD)
    return float(np.sqrt(np.sum((np.asarray(X, dtype=LD) - Xr) ** 2) / np.sum(Xr ** 2)))


# ---- CPU: the programs themselves and the oracle pinned to the reference ---------------------------------------------
def test_program_sizes():
    from george_b200._spec import flatten, num_params
    sizes = {"np8": 8, "np9": 9, "co2": 11, "np37": 37, "np64": 64, "np65": 65}
    for name, npar in sizes.items():
        assert num_params(flatten(_program(name))) == npar, name
    s = flatten(_program("leaves16"))
    assert s.n_nodes == 31 and sum(1 for i in range(s.n_nodes) if s.nodes[i].op == 0) == 16
    for name in ("depth8_1d", "depth8_3d"):
        s = flatten(_program(name))
        depth = top = 0
        for i in range(s.n_nodes):
            depth += 1 if s.nodes[i].op == 0 else -1
            top = max(top, depth)
        assert top == 8, (name, top)


def test_seventeen_leaves_do_not_fit():
    from george_b200._spec import flatten
    with pytest.raises(ValueError):
        flatten(_sixteen_leaves(extra=True))


def _reference_inputs(nd):
    rng = np.random.default_rng(3)
    return rng.normal(size=(23, nd)), rng.normal(size=(17, nd))


@pytest.mark.parametrize("name", NAMES)
def test_oracle_equals_reference_binary(oracle, name):
    import json
    from george_b200._spec import flatten
    from golden.make_golden_kernel_interface import PATH
    with open(PATH) as fh:
        ref = json.load(fh)
    kernel = _program(name)
    spec = flatten(kernel)
    x1, x2 = _reference_inputs(kernel.ndim)
    p = "limits__" + name + "__"
    assert golden_digest(oracle.value_general(spec, x1, x2)) == ref[p + "value_general"]
    assert golden_digest(oracle.value_symmetric(spec, x1)) == ref[p + "value_symmetric"]
    assert golden_digest(oracle.value_diagonal(spec, x1[:17], x2)) == ref[p + "value_diagonal"]
    which = np.ones(kernel.full_size, dtype=np.uint32)
    assert golden_digest(oracle.gradient_general(spec, which, x1, x2)) == ref[p + "gradient_general"]
    if kernel.ndim <= 8:
        assert golden_digest(oracle.x_gradient_general(spec, 1, x1, x2)) == ref[p + "x1_gradient_general"]
        assert golden_digest(oracle.x_gradient_general(spec, 2, x1, x2)) == ref[p + "x2_gradient_general"]


def reference_outputs(ref):
    """The reference's kernel_interface outputs that tests/golden/make_golden_kernel_interface.py digests."""
    out = {}
    for name, kernel in limit_programs():
        x1, x2 = _reference_inputs(kernel.ndim)
        r = ref.KernelInterface(kernel)
        p = "limits__" + name + "__"
        out[p + "value_general"] = r.value_general(x1, x2)
        out[p + "value_symmetric"] = r.value_symmetric(x1)
        out[p + "value_diagonal"] = r.value_diagonal(x1[:17], x2)
        out[p + "gradient_general"] = r.gradient_general(np.ones(kernel.full_size, dtype=np.uint32), x1, x2)
        if kernel.ndim <= 8:
            out[p + "x1_gradient_general"] = r.x1_gradient_general(x1, x2)
            out[p + "x2_gradient_general"] = r.x2_gradient_general(x1, x2)
    return out


# ---- GPU: evaluation ---------------------------------------------------------------------------------------------
def _points(n, nd, seed):
    return np.random.default_rng(seed).uniform(-2.0, 2.0, (n, nd))


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_values_match_oracle(gpu, oracle, record_property, name):
    from george_b200._spec import flatten
    kernel = _PROGRAMS[name]
    spec = flatten(kernel)
    rtol = VALUE_RTOL
    nd = kernel.ndim
    x1, x2 = _points(203, nd, 1), _points(131, nd, 2)
    errs = {"general": _err(kernel.get_value(x1, x2), oracle.value_general(spec, x1, x2), rtol, VALUE_ATOL)}
    ks = kernel.get_value(x1)
    assert np.array_equal(ks, ks.T)
    errs["symmetric"] = _err(ks, oracle.value_symmetric(spec, x1), rtol, VALUE_ATOL)
    errs["diagonal"] = _err(kernel.get_value(x1[:131], x2, diag=True), oracle.value_diagonal(spec, x1[:131], x2), rtol,
                            VALUE_ATOL)
    record_property("value_err", max(errs.values()))
    assert max(errs.values()) <= rtol, errs


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_matvec_matches_oracle(gpu, oracle, record_property, name):
    from george_b200._spec import flatten
    kernel = _PROGRAMS[name]
    spec = flatten(kernel)
    nd = kernel.ndim
    rng = np.random.default_rng(4)
    x1, x2 = _points(150, nd, 5), _points(600, nd, 6)  # 600 columns: two 512-column chunks
    K12 = oracle.value_general(spec, x1, x2).astype(LD)
    K22 = oracle.value_symmetric(spec, x2).astype(LD)
    worst = 0.0
    for nrhs in (1, 5):
        v = rng.standard_normal((600, nrhs))
        scale = np.abs(K12) @ np.abs(v.astype(LD))
        worst = max(worst, float(np.max(np.abs(kernel.matvec(x1, x2, v) - K12 @ v.astype(LD)) / scale)))
        d = rng.uniform(0.5, 1.0, 600)
        ref = K22 @ v.astype(LD) + d.astype(LD)[:, None] * v.astype(LD)
        scale = np.abs(K22) @ np.abs(v.astype(LD)) + (d[:, None] * np.abs(v)).astype(LD)
        worst = max(worst, float(np.max(np.abs(kernel.matvec(x2, x2, v, diag=d) - ref) / scale)))
    v1 = rng.standard_normal(600)
    out = kernel.matvec(x1, x2, v1)
    assert out.shape == (150,)
    worst = max(worst, float(np.max(np.abs(out - K12 @ v1.astype(LD)) / (np.abs(K12) @ np.abs(v1.astype(LD))))))
    record_property("matvec_err", worst)
    assert worst <= MATVEC_TOL, worst


@pytest.mark.gpu
@pytest.mark.parametrize("name", GRAD_NAMES)
def test_gradients_match_oracle(gpu, oracle, record_property, name):
    from george_b200._spec import flatten
    kernel = _PROGRAMS[name]
    spec = flatten(kernel)
    nd = kernel.ndim
    x1, x2 = _points(37, nd, 7), _points(29, nd, 8)
    which = np.ones(kernel.full_size, dtype=np.uint32)
    errs = [_err(kernel.get_gradient(x1, x2, include_frozen=True), oracle.gradient_general(spec, which, x1, x2),
                 GRAD_RTOL, GRAD_ATOL),
            _err(kernel.get_gradient(x1, include_frozen=True), oracle.gradient_general(spec, which, x1, x1),
                 GRAD_RTOL, GRAD_ATOL)]
    record_property("grad_err", max(errs))
    assert max(errs) <= GRAD_RTOL, errs


@pytest.mark.gpu
@pytest.mark.parametrize("name", XGRAD_NAMES)
def test_x_gradients_match_oracle(gpu, oracle, record_property, name):
    from george_b200._spec import flatten
    kernel = _PROGRAMS[name]
    spec = flatten(kernel)
    nd = kernel.ndim
    x1, x2 = _points(37, nd, 9), _points(29, nd, 10)
    errs = [_err(kernel.get_x1_gradient(x1, x2), oracle.x_gradient_general(spec, 1, x1, x2), GRAD_RTOL, GRAD_ATOL),
            _err(kernel.get_x2_gradient(x1, x2), oracle.x_gradient_general(spec, 2, x1, x2), GRAD_RTOL, GRAD_ATOL)]
    record_property("xgrad_err", max(errs))
    assert max(errs) <= GRAD_RTOL, errs


@pytest.mark.gpu
def test_expression_deeper_than_the_interpreter_stack_is_rejected(gpu):
    d1 = _depth_1d_leaves()
    k = _right_nested(d1, ["+"] * 8)
    x = np.linspace(0, 1, 5)[:, None]
    with pytest.raises(ValueError, match="too deep"):
        k.get_value(x)
    assert np.all(np.isfinite(_right_nested(d1[:8], ["+"] * 7).get_value(x)))


@pytest.mark.gpu
@pytest.mark.parametrize("n", CONTRACT_N)
@pytest.mark.parametrize("name", CONTRACT_NAMES)
def test_gradient_contraction_against_extended_precision(gpu, oracle, record_property, name, n):
    """g = sum_ij A_ij dK_ij for a non-symmetric A, with the first, a middle and the last parameter frozen."""
    from george_b200._spec import flatten
    kernel = _PROGRAMS[name]
    spec = flatten(kernel)
    npar = kernel.full_size
    rng = np.random.default_rng(n)
    x = _points(n, kernel.ndim, 11 + n)
    A = rng.standard_normal((n, n))
    which = np.ones(npar, dtype=np.uint32)
    frozen = [0, npar // 2, npar - 1]
    which[frozen] = 0
    g = kernel.kernel.gradient_contract(which, x, A)
    dK = oracle.gradient_general(spec, np.ones(npar, dtype=np.uint32), x, x).astype(LD)
    g_ref = np.einsum("ijk,ij->k", dK, A.astype(LD))
    scale = np.einsum("ijk,ij->k", np.abs(dK), np.abs(A).astype(LD))
    live = which.astype(bool)
    assert np.all(g[frozen] == 0.0)
    err = float(np.max(np.abs(g[live] - g_ref[live]) / np.maximum(scale[live], LD(1e-300))))
    record_property("contract_err", err)
    assert err <= CONTRACT_TOL, err


# ---- GPU: solvers ------------------------------------------------------------------------------------------------
class _Problem(object):
    """K = oracle K(x, x) + diag(sig^2) and everything the solver tests compare with, in longdouble."""

    def __init__(self, kernel, x, sig, r, xs, oracle, inverse=True):
        from george_b200._spec import flatten
        spec = flatten(kernel)
        self.kernel, self.x, self.sig, self.r, self.xs = kernel, x, sig, r, xs
        n = len(x)
        K = oracle.value_symmetric(spec, x)
        K[np.diag_indices(n)] += sig * sig
        self.cond = np.linalg.cond(K)
        self.L = hiprec.chol_ld(K)
        self.logdet = hiprec.logdet_ld(self.L)
        self.alpha = hiprec.solve_ld(self.L, r)
        Kxs = oracle.value_general(spec, xs, x).astype(LD)
        self.mean = Kxs @ self.alpha
        self.mean_scale = np.abs(Kxs) @ np.abs(self.alpha)
        W = np.array(Kxs.T)
        for i in range(n):  # W = L^-1 K(x, x*)
            W[i] = (W[i] - self.L[i, :i] @ W[:i]) / self.L[i, i]
        self.kss = oracle.value_symmetric(spec, xs)
        self.cov = self.kss.astype(LD) - W.T @ W
        self.var = np.diag(self.cov)
        if inverse:
            self.Kinv = hiprec.solve_ld(self.L, np.eye(n))
            which = np.ones(kernel.full_size, dtype=np.uint32)
            self.dK = oracle.gradient_general(spec, which, x, x).astype(LD)


_CACHE = {}


def _solver_problem(name, oracle):
    if name not in _CACHE:
        from george_b200 import kernels as K
        n, inverse = 300, True
        if name == "co2":  # the tutorial's kernel with a unit long-term amplitude: cond(K) <= 1e4
            kernel = _co2_kernel(1.0)
            x = np.sort(np.random.default_rng(12).uniform(1958, 2003, n))[:, None]
        elif name == "leaves16_768":  # two 768-row HODLR leaves; points on a curve keep the off-diagonal block low rank
            n, inverse = 1536, False
            kernel = _sixteen_leaves()
            t = np.sort(np.random.default_rng(13).uniform(-2, 2, n))
            x = np.stack([t, 0.5 * np.sin(2 * t), 0.3 * t * t], axis=1)
        else:
            kernel = _program(name) if name in _PROGRAMS else wide_kernel(int(name[5:-1]))
            x = _points(n, kernel.ndim, 14)
        rng = np.random.default_rng(15)
        sig = 0.6 + 0.4 * rng.uniform(size=n)
        if name == "leaves16_768":
            sig = sig + 0.9
        r = rng.standard_normal(n)
        lo, hi = x.min(axis=0), x.max(axis=0)
        xs = lo + (hi - lo) * rng.uniform(size=(40, x.shape[1]))
        _CACHE[name] = _Problem(kernel, x, sig, r, xs, oracle, inverse)
        assert _CACHE[name].cond <= 1e4, (name, _CACHE[name].cond)
    return _CACHE[name]


def _hodlr(kernel, rng_mode, min_size=50):
    import george_b200 as george
    return george.HODLRSolver(kernel, min_size=min_size, tol=1e-15, seed=42, rng_mode=rng_mode, exhaust="dense")


def _check_solver(s, P, record_property, tol, grad=True):
    import george_b200 as george
    s.compute(P.x, P.sig)
    errs = {"logdet": abs(float(s.log_determinant - P.logdet)) / max(1.0, abs(float(P.logdet))),
            "solve": _rel(np.ravel(s.apply_inverse(P.r)), P.alpha)}
    B = np.stack([P.r, np.cos(P.r), P.r ** 2], axis=1)
    errs["solve3"] = _rel(s.apply_inverse(B), hiprec.solve_ld(P.L, B))
    scale = float(np.max(np.abs(P.kss)))
    mean = P.kernel.matvec(P.xs, P.x, np.ravel(s.apply_inverse(P.r)))
    errs["mean"] = float(np.max(np.abs(mean - P.mean) / P.mean_scale))
    errs["var"] = float(np.max(np.abs(s.predictive(P.kernel, P.xs, "var") - P.var))) / scale
    errs["cov"] = float(np.max(np.abs(s.predictive(P.kernel, P.xs, "cov") - P.cov))) / scale
    # GP.predict on the same factorisation (its mean is the matvec above plus a zero mean)
    gp = george.GP(P.kernel)
    gp.compute(P.x, P.sig)
    gp.solver = s
    mu, cov = gp.predict(P.r, P.xs)
    errs["gp_mean"] = float(np.max(np.abs(mu - P.mean) / P.mean_scale))
    errs["gp_cov"] = float(np.max(np.abs(cov - P.cov))) / scale
    if grad:
        which = np.ones(P.kernel.full_size, dtype=np.uint32)
        alpha, g, dA = s.grad_terms(P.r, which)
        Amat = np.outer(P.alpha, P.alpha) - P.Kinv
        g_ref = np.einsum("ijk,ij->k", P.dK, Amat)
        g_scale = np.einsum("ijk,ij->k", np.abs(P.dK), np.abs(Amat))
        errs["grad_alpha"] = _rel(alpha, P.alpha)
        errs["grad_g"] = float(np.max(np.abs(g - g_ref) / g_scale))
        errs["grad_diag"] = _rel(dA, np.diag(Amat))
    for k, v in errs.items():
        record_property(k + "_err", v)
    assert errs["logdet"] <= tol["logdet"], errs
    assert max(errs["solve"], errs["solve3"]) <= tol["solve"], errs
    assert max(errs["mean"], errs["var"], errs["cov"], errs["gp_mean"], errs["gp_cov"]) <= tol["predict"], errs
    if grad:
        assert max(errs["grad_alpha"], errs["grad_g"], errs["grad_diag"]) <= tol["grad"], errs


DENSE_PROBLEMS = ["np64", "co2", "depth8_1d", "depth8_3d", "leaves16",
                  "wide_8d", "wide_29d", "wide_32d", "wide_56d", "wide_59d", "wide_100d"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", DENSE_PROBLEMS)
def test_basic_solver_against_extended_precision(gpu, oracle, record_property, name):
    import george_b200 as george
    P = _solver_problem(name, oracle)
    _check_solver(george.BasicSolver(P.kernel), P, record_property, DENSE_TOL, grad=len(P.kernel) <= 64)


@pytest.mark.gpu
@pytest.mark.parametrize("rng_mode", ["pernode", "reference"])
@pytest.mark.parametrize("name", ["np64", "co2", "leaves16", "wide_29d", "wide_32d"])
def test_hodlr_solver_against_extended_precision(gpu, oracle, record_property, name, rng_mode):
    P = _solver_problem(name, oracle)
    _check_solver(_hodlr(P.kernel, rng_mode), P, record_property, HODLR_TOL)


@pytest.mark.gpu
def test_hodlr_rejects_33_dimensions(gpu):
    k = wide_kernel(33)
    x = _points(200, 33, 16)
    with pytest.raises(ValueError, match="32"):
        _hodlr(k, "pernode").compute(x, np.full(200, 0.5))


@pytest.mark.gpu
@pytest.mark.parametrize("rng_mode", ["pernode", "reference"])
def test_hodlr_sixteen_leaves_at_the_largest_leaf(gpu, oracle, record_property, rng_mode):
    """n = 1536, min_size = 768: two 768-row leaves, the staged 16-leaf program in the generic leaf factorisation."""
    P = _solver_problem("leaves16_768", oracle)
    s = _hodlr(P.kernel, rng_mode, min_size=768)
    s.compute(P.x, P.sig)
    assert [nd["size"] for nd in s.solver.nodes() if nd["is_leaf"]] == [768, 768]
    errs = {"logdet": abs(float(s.log_determinant - P.logdet)) / max(1.0, abs(float(P.logdet))),
            "solve": _rel(np.ravel(s.apply_inverse(P.r)), P.alpha)}
    scale = float(np.max(np.abs(P.kss)))
    errs["var"] = float(np.max(np.abs(s.predictive(P.kernel, P.xs, "var") - P.var))) / scale
    for k, v in errs.items():
        record_property(k + "_err", v)
    assert (errs["logdet"] <= HODLR_TOL["logdet"] and errs["solve"] <= HODLR_TOL["solve"]
            and errs["var"] <= HODLR_TOL["predict"]), errs


def _fitted_gp(kernel, solver, x, y, **kw):
    import george_b200 as george
    gp = george.GP(kernel, mean=float(np.mean(y)), fit_mean=True, white_noise=np.log(0.5 ** 2), fit_white_noise=True,
                   solver=solver, **kw)
    gp.compute(x)
    return gp


def _grad_ll_reference(gp, y, oracle):
    """GP.grad_log_likelihood (mean, white noise, kernel) from the longdouble K^-1; and the scale of each entry."""
    from george_b200._spec import flatten
    x = gp._x
    sig = gp._sigma(x)
    K = oracle.value_symmetric(flatten(gp.kernel), x)
    K[np.diag_indices(len(x))] += sig * sig
    assert np.linalg.cond(K) <= 1e4
    L = hiprec.chol_ld(K)
    alpha = hiprec.solve_ld(L, y - gp._call_mean(x))
    A = np.outer(alpha, alpha) - hiprec.solve_ld(L, np.eye(len(x)))
    dK = oracle.gradient_general(flatten(gp.kernel), np.ones(gp.kernel.full_size, dtype=np.uint32), x, x).astype(LD)
    wn = np.exp(gp._call_white_noise(x)).astype(LD)
    ref = [np.sum(alpha), 0.5 * np.sum(wn * np.diag(A))] + list(0.5 * np.einsum("ijk,ij->k", dK, A))
    scale = [np.sum(np.abs(alpha)), 0.5 * np.sum(wn * np.abs(np.diag(A)))] + list(
        0.5 * np.einsum("ijk,ij->k", np.abs(dK), np.abs(A)))
    return np.array(ref, dtype=LD), np.array(scale, dtype=LD)


@pytest.mark.gpu
@pytest.mark.parametrize("solver_name", ["basic", "hodlr"])
@pytest.mark.parametrize("name", ["co2", "np64"])
def test_grad_log_likelihood_fitted_mean_and_white_noise(gpu, oracle, record_property, name, solver_name):
    import george_b200 as george
    if name == "co2":
        kernel = _co2_kernel(1.0)
        rng = np.random.default_rng(17)
        x = np.sort(rng.uniform(1958, 2003, 300))
        y = 315 + 1.3 * (x - 1958) + 3 * np.sin(2 * np.pi * x) + 0.3 * rng.standard_normal(300)
    else:
        kernel = _np64_kernel()
        x = _points(300, 8, 18)
        y = np.sin(x[:, 0]) * np.cos(x[:, 3]) + 0.3 * np.random.default_rng(19).standard_normal(300)
    kw = {} if solver_name == "basic" else dict(min_size=50, tol=1e-15, rng_mode="pernode", exhaust="dense")
    gp = _fitted_gp(kernel, george.BasicSolver if solver_name == "basic" else george.HODLRSolver, x, y, **kw)
    g = gp.grad_log_likelihood(y)
    assert len(g) == 2 + kernel.full_size
    ref, scale = _grad_ll_reference(gp, y, oracle)
    err = float(np.max(np.abs(g - ref) / scale))
    record_property("grad_ll_err", err)
    assert err <= (DENSE_TOL if solver_name == "basic" else HODLR_TOL)["grad"], err


@pytest.mark.gpu
@pytest.mark.parametrize("solver_name", ["basic", "hodlr"])
def test_65_parameters_are_rejected_before_anything_is_solved(gpu, solver_name):
    import george_b200 as george
    kernel = _np64_kernel(5)
    x = _points(200, 8, 20)
    y = np.sin(x[:, 0])
    which = np.ones(65, dtype=np.uint32)
    with pytest.raises(ValueError, match="64"):
        kernel.get_gradient(x)
    with pytest.raises(ValueError, match="64"):
        kernel.kernel.gradient_contract(which, x, np.eye(200))
    kw = {} if solver_name == "basic" else dict(min_size=50, tol=1e-15, rng_mode="pernode", exhaust="dense")
    gp = _fitted_gp(kernel, george.BasicSolver if solver_name == "basic" else george.HODLRSolver, x, y, **kw)
    ll0 = gp.log_likelihood(y)
    with pytest.raises(ValueError, match="64"):
        gp.solver.grad_terms(y - np.mean(y), which)
    with pytest.raises(ValueError, match="64"):
        gp.grad_log_likelihood(y)
    assert gp.log_likelihood(y) == ll0
    assert np.all(gp.grad_log_likelihood(y, quiet=True) == 0.0)


# ---- GPU: batches ------------------------------------------------------------------------------------------------
def _single(kernel, p, x, sig, r, xs, what):
    from george_b200 import BasicSolver
    p0 = kernel.get_parameter_vector(include_frozen=True)
    kernel.set_parameter_vector(p, include_frozen=True)
    try:
        s = BasicSolver(kernel)
        s.compute(x, sig)
        alpha = s.apply_inverse(np.array(r), in_place=True).flatten()
        return s.log_determinant, s.dot_solve(r), kernel.matvec(xs, x, alpha), (s.predictive(kernel, xs, what) if what else None)
    finally:
        kernel.set_parameter_vector(p0, include_frozen=True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["np64", "leaves16", "wide_29d", "wide_59d", "wide_100d"])
def test_batches_match_the_single_path(gpu, oracle, record_property, name):
    from george_b200 import BasicSolver
    from george_b200._spec import flatten
    kernel = _program(name) if name in _PROGRAMS else wide_kernel(int(name[5:-1]))
    spec = flatten(kernel)
    n, nb = 200, 3
    rng = np.random.default_rng(21)
    x = _points(n, kernel.ndim, 22)
    xs = _points(9, kernel.ndim, 23)
    p0 = kernel.get_parameter_vector(include_frozen=True)
    params = p0 + 0.02 * rng.standard_normal((nb, len(p0)))
    sig = 0.6 + 0.4 * rng.uniform(size=(nb, n))
    r = rng.standard_normal((nb, n))
    ld, q, info = BasicSolver.batch_log_likelihood(spec, params, x, sig, r)
    assert np.all(info == 0)
    worst = {"logdet": 0.0, "dot": 0.0}
    for what in (None, "var", "cov"):
        mean, out, info = BasicSolver.batch_predict(spec, params, x, sig, r, xs, what)
        assert np.all(info == 0)
        for b in range(nb):
            ld1, q1, m1, o1 = _single(kernel, params[b], x, sig[b], r[b], xs, what)
            assert ld[b] == ld1 and abs(q[b] - q1) <= 1e-13 * abs(q1), (b, ld[b], ld1, q[b], q1)
            assert np.array_equal(mean[b], m1), (what, b)
            if what is not None:
                assert np.array_equal(out[b], o1), (what, b)
    try:
        for b in range(nb):
            kernel.set_parameter_vector(params[b], include_frozen=True)
            K = oracle.value_symmetric(flatten(kernel), x)
            K[np.diag_indices(n)] += sig[b] * sig[b]
            assert np.linalg.cond(K) <= 1e4
            L = hiprec.chol_ld(K)
            ref_ld = hiprec.logdet_ld(L)
            ref_q = np.dot(r[b].astype(LD), hiprec.solve_ld(L, r[b]))
            worst["logdet"] = max(worst["logdet"], abs(float(ld[b] - ref_ld)) / max(1.0, abs(float(ref_ld))))
            worst["dot"] = max(worst["dot"], abs(float(q[b] - ref_q)) / abs(float(ref_q)))
    finally:
        kernel.set_parameter_vector(p0, include_frozen=True)
    record_property("logdet_err", worst["logdet"])
    record_property("dot_err", worst["dot"])
    assert worst["logdet"] <= DENSE_TOL["logdet"] and worst["dot"] <= DOT_TOL, worst
