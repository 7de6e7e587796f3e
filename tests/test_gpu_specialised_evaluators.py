# -*- coding: utf-8 -*-
"""The specialised kernel evaluators against the postfix interpreter, bit for bit.

Two families of evaluators stand in for the interpreter (`kernel_value`, csrc/kernel_eval.cuh) when a program has a
known structure: the kernel-matrix builds' `ProfileND<SHAPE, ND, AXIS>` (csrc/kmat.cu, `detect_fast_shape`) and the 1-D
program shapes' `ScaledProfile1D<SHAPE>` (shape set in csrc/core.cu; the ACA, the HODLR leaves, the matvec).  Both
promise the interpreter's arithmetic in the interpreter's order.  `bgp_spec_paths` tells which evaluator a program gets;
FORMS below pins that choice for every program form, and the GPU tests compare each specialised route with its
*generic twin*: the same kernel times a constant kernel of value exactly 1.0.  That product is exact, so the twin's
values are the interpreter's values of the same program, and its extra node defeats every detection rule.  1-D programs
are embedded in 2-D for the twin (`ndim=2, axes=0`, second coordinate 0) so that the general interpreter runs, not its
1-D shortcut; the shortcut is checked against the specialised route as well.

The input-gradient evaluator of the one-term shapes (`ScaledProfileGrad1D`, GP.grad_predict) multiplies in another
order than the interpreter; both are held to a few ulp of an mpmath reference instead.
"""
import ctypes as C
import math

import numpy as np
import pytest

from george_b200 import kernels as K

EPS = np.finfo(np.float64).eps

# csrc/kernel_eval.cuh BGP_SHAPE_*
EXPSQ, M32, M52, EXP, SUM_EXPSQ, SUM_M32, PROD_EXPSQ, PROD_M32 = range(1, 9)
PROFILES = {"expsq": (K.ExpSquaredKernel, EXPSQ), "m32": (K.Matern32Kernel, M32),
            "m52": (K.Matern52Kernel, M52), "exp": (K.ExpKernel, EXP)}
# r2 above which profile_value returns 0 without evaluating exp
CUTOFF = {"expsq": 1490.4, "m32": 185200.0, "m52": 111100.0, "exp": 555400.0}
AXIS_METRIC = [0.7, 1.9, 0.45]
ISO_METRIC = 1.3
LOG_C, LOG_C2 = math.log(1.7), math.log(0.6)


def _leaf(prof, nd, axis, ndim, axes):
    cls = PROFILES[prof][0]
    return cls(metric=AXIS_METRIC[:nd] if axis else ISO_METRIC, ndim=ndim, axes=axes)


def _const(log_c, ndim, axes):
    return K.ConstantKernel(log_constant=log_c, ndim=ndim, axes=axes)


def _es2(ndim, axes, gamma=1.3):
    return K.ExpSine2Kernel(gamma=gamma, log_period=math.log(2.7), ndim=ndim, axes=axes)


class Form(object):
    """A program form: build(ndim, axes) makes it on `nd` input dimensions (ndim=2, axes=[0] embeds a 1-D form in 2-D);
    want = (1-D program shape, FAST1D flag, kmat profile, kmat ND, kmat axis-aligned) of bgp_spec_paths."""

    def __init__(self, name, nd, build, want):
        self.name, self.nd, self.build, self.want = name, nd, build, tuple(want)

    def kernel(self):
        return self.build(self.nd, None)

    def twin(self, embed=True):
        """the form times ConstantKernel(log_constant=0) on one axis: the interpreter's values, bit for bit"""
        if self.nd == 1 and embed:
            ndim, axes = 2, [0]
        else:
            ndim, axes = self.nd, None
        from george_b200._spec import flatten
        one = _const(0.0, ndim, [0])
        assert len(one.axes) == 1 and math.exp(one.get_parameter_vector(include_frozen=True)[0]) == 1.0
        base = self.build(ndim, axes)
        if flatten(base).n_nodes == 1:  # [S, 1, *] is itself the form S * c: one more factor
            base = base * _const(0.0, ndim, [0])
        return base * one

    def __repr__(self):
        return self.name


def _one_term_forms():
    out = []
    for prof, (_, shape) in PROFILES.items():
        for nd in (1, 2, 3):
            for axis in (False, True):
                want = (shape if nd == 1 else 0, 1 if nd == 1 else 0, shape, nd, int(axis))
                tag = "{0}_{1}d_{2}".format(prof, nd, "axis" if axis else "iso")

                def S(ndim, axes, p=prof, n=nd, a=axis):
                    return _leaf(p, n, a, ndim, axes)
                out.append(Form(tag + "_S", nd, S, want))
                # the constant spans every axis of the form: its value is summed over them
                out.append(Form(tag + "_cS", nd, lambda ndim, axes, S=S: _const(LOG_C, ndim, axes) * S(ndim, axes),
                                want))
                out.append(Form(tag + "_Sc", nd, lambda ndim, axes, S=S: S(ndim, axes) * _const(LOG_C, ndim, axes),
                                want))
    return out


def _two_term_forms():
    out = []
    for prof, sum_shape, prod_shape in (("expsq", SUM_EXPSQ, PROD_EXPSQ), ("m32", SUM_M32, PROD_M32)):
        def S(ndim, axes, p=prof):
            return _leaf(p, 1, False, ndim, axes)

        def cS(ndim, axes, S=S):
            return _const(LOG_C, ndim, axes) * S(ndim, axes)

        def c2E(ndim, axes):
            return _const(LOG_C2, ndim, axes) * _es2(ndim, axes)

        want_sum, want_prod = (sum_shape, 1, 0, 0, 0), (prod_shape, 1, 0, 0, 0)
        out += [
            Form(prof + "_cS+c2E", 1, lambda nd_, ax, cS=cS: cS(nd_, ax) + c2E(nd_, ax), want_sum),
            Form(prof + "_c2E+cS", 1, lambda nd_, ax, cS=cS: c2E(nd_, ax) + cS(nd_, ax), want_sum),
            Form(prof + "_Ec2+Sc", 1, lambda nd_, ax, S=S: _es2(nd_, ax) * _const(LOG_C2, nd_, ax)
                 + S(nd_, ax) * _const(LOG_C, nd_, ax), want_sum),
            Form(prof + "_S+E", 1, lambda nd_, ax, S=S: S(nd_, ax) + _es2(nd_, ax), want_sum),
            Form(prof + "_cS*E", 1, lambda nd_, ax, cS=cS: cS(nd_, ax) * _es2(nd_, ax), want_prod),
            Form(prof + "_S*E", 1, lambda nd_, ax, S=S: S(nd_, ax) * _es2(nd_, ax), want_prod),
            # exp(-Gamma sin^2) > 1 for Gamma < 0
            Form(prof + "_cS*E_neg_gamma", 1, lambda nd_, ax, cS=cS: cS(nd_, ax) * _es2(nd_, ax, gamma=-0.7), want_prod),
        ]
    return out


def _interpreter_forms():
    """forms that no detection rule may take (build ignores its arguments: these have no twin)"""
    def S(prof="expsq", ndim=1, axes=None, **kw):
        return PROFILES[prof][0](metric=ISO_METRIC, ndim=ndim, axes=axes, **kw)

    def E():
        return _es2(1, None)

    c, c2 = math.exp(LOG_C), math.exp(LOG_C2)
    fast1d, none = (0, 1, 0, 0, 0), (0, 0, 0, 0, 0)
    table = [
        ("E*S", 1, lambda: E() * S(), fast1d),
        ("(c*E)*S", 1, lambda: (c2 * E()) * S(), fast1d),        # rounds differently from (c*S)*E
        ("c*(S*E)", 1, lambda: c * (S() * E()), fast1d),
        ("m52_cS+c2E", 1, lambda: c * S("m52") + c2 * E(), fast1d),
        ("exp_cS+c2E", 1, lambda: c * S("exp") + c2 * E(), fast1d),
        ("m52_cS*E", 1, lambda: c * S("m52") * E(), fast1d),
        ("exp_cS*E", 1, lambda: c * S("exp") * E(), fast1d),
        ("axes_permuted", 2, lambda: K.ExpSquaredKernel(metric=[0.7, 1.9], ndim=2, axes=[1, 0]), none),
        ("axes_subset", 3, lambda: c * S("m32", ndim=3, axes=[0, 2]), none),
        ("blocked", 1, lambda: c * S(block=[(-1e9, 1e9)]), none),
        ("general_metric", 2, lambda: K.ExpSquaredKernel([[1.0, 0.2], [0.2, 1.5]], ndim=2), none),
        ("ratquad", 1, lambda: c * K.RationalQuadraticKernel(log_alpha=0.3, metric=ISO_METRIC), fast1d),
        ("user_cauchy", 1, lambda: c * K.CauchyKernel(metric=ISO_METRIC), none),
        ("expsq_4d", 4, lambda: c * S(ndim=4), none),
        ("expsq+m32", 1, lambda: S() + S("m32"), fast1d),
    ]
    return [Form(name, nd, lambda ndim, axes, mk=mk: mk(), want) for name, nd, mk, want in table]


ONE_TERM = _one_term_forms()
TWO_TERM = _two_term_forms()
SPECIALISED = ONE_TERM + TWO_TERM
FORMS = SPECIALISED + _interpreter_forms()


def spec_paths(kernel):
    from george_b200 import _lib
    from george_b200._spec import flatten
    spec = flatten(kernel)
    out = (C.c_int32 * 5)()
    _lib.check(_lib.load().bgp_spec_paths(C.byref(spec), out))
    return tuple(out)


# ---- host: the evaluator each form gets ------------------------------------------------------------------------------

@pytest.mark.parametrize("form", FORMS, ids=repr)
def test_each_form_takes_the_path_it_names(form):
    assert spec_paths(form.kernel()) == form.want
    if form in SPECIALISED:  # the twins run on the interpreter, the embedded one without its 1-D shortcut
        assert spec_paths(form.twin()) == (0, 0, 0, 0, 0)
        if form.nd == 1:
            assert spec_paths(form.twin(embed=False)) == (0, 1, 0, 0, 0)


def test_spec_paths_rejects_an_invalid_program():
    from george_b200 import _lib
    from george_b200._spec import flatten
    spec = flatten(K.ExpSquaredKernel(1.0))
    spec.nodes[0].kernel_type = 99
    out = (C.c_int32 * 5)()
    assert _lib.load().bgp_spec_paths(C.byref(spec), out) == _lib.BGP_ERR_INVALID


# ---- helpers of the GPU tests ------------------------------------------------------------------------------------------

def assert_bits_equal(a, b, what=""):
    """same float64 bits everywhere, NaN matching NaN"""
    a, b = np.ascontiguousarray(a, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64)
    assert a.shape == b.shape, what
    na, nb = np.isnan(a), np.isnan(b)
    assert np.array_equal(na, nb), what
    ia, ib = a.view(np.int64)[~na], b.view(np.int64)[~nb]
    bad = np.flatnonzero(ia != ib)
    assert bad.size == 0, "{0}: {1} of {2} entries differ, first {3!r} vs {4!r}".format(
        what, bad.size, ia.size, a[~na][bad[0]], b[~nb][bad[0]])


def _embed(x):
    """1-D points as 2-D points with a zero second coordinate"""
    x = np.asarray(x, dtype=np.float64).reshape(len(x), -1)
    return np.ascontiguousarray(np.column_stack([x, np.zeros(len(x))]))


def _coords(n, nd, seed):
    """points near 2.45e6 with a spread of a few length scales, and exact duplicates (r2 = 0)"""
    rng = np.random.default_rng(seed)
    x = 2.45e6 + rng.uniform(0.0, 2.0 + n / 40.0, (n, nd))
    if n > 3:
        x[1::5] = x[0:n - 1:5][:len(x[1::5])]
    return np.ascontiguousarray(x)


def _routes(form, x):
    """(specialised kernel, its input), then the interpreter twins with theirs"""
    out = [(form.kernel(), x), (form.twin(), _embed(x) if form.nd == 1 else x)]
    if form.nd == 1:
        out.append((form.twin(embed=False), x))
    return out


SIZES = [1, 63, 64, 65, 127, 128, 129, 200]


@pytest.mark.gpu
@pytest.mark.parametrize("form", SPECIALISED, ids=repr)
def test_kernel_matrix_builds_match_the_interpreter(gpu, form):
    """get_value (general, symmetric, diagonal) of the specialised route against its twins, on and around the tiles'
    edges (64-row / 128-column tiles)."""
    for i, n in enumerate(SIZES):
        x1 = _coords(n, form.nd, 10 + i)
        x2 = _coords(SIZES[(i + 3) % len(SIZES)], form.nd, 40 + i)
        got = []
        for kern, emb in _routes(form, x1):
            x2r = _embed(x2) if emb.shape[1] != x2.shape[1] else x2
            got.append((kern.get_value(emb, x2r), kern.get_value(emb), kern.get_value(emb, diag=True)))
        for route in got[1:]:
            for a, b, what in zip(got[0], route, ("general", "symmetric", "diagonal")):
                assert_bits_equal(a, b, "{0} n={1}".format(what, n))


def _params(kernel, twin, B, seed):
    """B parameter vectors differing in every constant and metric parameter; the twin's extra constants stay 0"""
    from george_b200._spec import flatten, num_params
    p0 = np.asarray(kernel.get_parameter_vector(include_frozen=True), dtype=np.float64)
    extra = num_params(flatten(twin)) - p0.size
    assert num_params(flatten(kernel)) == p0.size and extra in (1, 2)
    rng = np.random.default_rng(seed)
    p = p0[None, :] + rng.uniform(-0.4, 0.4, (B, p0.size))
    p[0] = p0
    return p, np.column_stack([p, np.zeros((B, extra))])


@pytest.mark.gpu
@pytest.mark.parametrize("form", SPECIALISED, ids=repr)
def test_dense_solver_and_batches_match_the_interpreter(gpu, form):
    """BasicSolver.compute's K + diag(yerr^2) (the build it runs, on the device), its log-determinant and solve, and
    batch_log_likelihood / batch_predict with members that differ in every parameter."""
    import torch
    from george_b200 import _lib
    from george_b200._spec import flatten
    from george_b200.solvers.basic import BasicSolver
    lib = _lib.load()
    B = 3
    for n in (65, 129, 200):
        x = _coords(n, form.nd, n)
        xs = _coords(70, form.nd, n + 1)
        rng = np.random.default_rng(n)
        yerr = 0.3 + rng.uniform(0, 0.2, n)
        r = rng.normal(size=(B, n))
        res = []
        for kern, emb in _routes(form, x)[:2]:
            spec = flatten(kern)
            xd = torch.tensor(emb, dtype=torch.float64, device="cuda")
            dd = torch.tensor(yerr ** 2, dtype=torch.float64, device="cuda")
            Kd = torch.empty((n, n), dtype=torch.float64, device="cuda")
            torch.cuda.synchronize()
            _lib.check(lib.bgp_kmat_symmetric_dev(C.byref(spec), C.c_void_p(xd.data_ptr()), n,
                                                  C.c_void_p(dd.data_ptr()), C.c_void_p(Kd.data_ptr()), n))
            torch.cuda.synchronize()
            res.append({"K": Kd.cpu().numpy()})
            s = BasicSolver(kern)
            try:  # (c*S)*ExpSine2 with Gamma < 0 need not be positive definite: both routes fail alike then
                s.compute(emb, yerr)
                res[-1].update(logdet=s.log_determinant, solve=s.apply_inverse(r[0]))
            except np.linalg.LinAlgError as e:
                res[-1].update(logdet=np.nan, solve=np.full(n, np.nan), error=str(e))
        assert res[0].get("error") == res[1].get("error")
        p_spec, p_twin = _params(form.kernel(), form.twin(), B, n)
        for (kern, emb), p, out in zip(_routes(form, x)[:2], (p_spec, p_twin), res):
            xse = _embed(xs) if emb.shape[1] != xs.shape[1] else xs
            spec = flatten(kern)
            yb = np.tile(yerr, (B, 1))
            ld, quad, info = BasicSolver.batch_log_likelihood(spec, p, emb, yb, r)
            mean, var, info2 = BasicSolver.batch_predict(spec, p, emb, yb, r, xse, "var")
            assert np.array_equal(info, info2)
            out.update(batch_logdet=ld, batch_quad=quad, batch_mean=mean, batch_var=var, info=info)
        assert np.array_equal(res[0]["info"], res[1]["info"])
        if "neg_gamma" not in form.name:
            assert "error" not in res[0] and np.all(res[0]["info"] == 0)
        for key in ("K", "logdet", "solve", "batch_logdet", "batch_quad", "batch_mean", "batch_var"):
            assert_bits_equal(res[0][key], res[1][key], "{0} n={1}".format(key, n))


ONE_TERM_1D = [f for f in ONE_TERM if f.nd == 1]


@pytest.mark.gpu
@pytest.mark.parametrize("form", ONE_TERM_1D, ids=repr)
def test_matvec_matches_the_interpreter(gpu, form):
    """kernel.matvec (bgp_kmat_matvec, ScaledProfile1D in its tiles) with random right-hand sides"""
    for n1, n2 in ((1, 1), (63, 129), (200, 300), (129, 1000)):
        x1, x2 = _coords(n1, 1, n1), _coords(n2, 1, n2 + 7)
        v = np.random.default_rng(n1 + n2).normal(size=(n2, 3))
        got = [k.matvec(a, _embed(x2) if a.shape[1] == 2 else x2, v) for k, a in _routes(form, x1)]
        for g in got[1:]:
            assert_bits_equal(got[0], g, "matvec {0}x{1}".format(n1, n2))


def _sweep_r2(prof):
    """r2 across the profile's cutoff (relative +-1e-3) and where exp of the profile's argument is subnormal"""
    cut = CUTOFF[prof]
    a = np.linspace(708.5, 745.5, 1500)  # exponent argument a: exp(-a) in the subnormal range and past 0
    r2_sub = {"expsq": 2 * a, "m32": a * a / 3, "m52": a * a / 5, "exp": a * a}[prof]
    return np.r_[np.linspace(cut * (1 - 1e-3), cut * (1 + 1e-3), 3000), r2_sub]


@pytest.mark.gpu
@pytest.mark.parametrize("prof", list(PROFILES))
def test_far_field_cutoff_agrees_with_device_exp(gpu, record_property, prof):
    """One-hot right-hand sides extract single entries exactly (only +0 terms are added): with m = 1 and x2 = 0 the
    entries k(x1, 0) of the specialised matvec, whose profile_value returns 0 past the cutoff, against the interpreter's
    exp across the cutoff and through the subnormal range.  A nonzero subnormal from the interpreter past the cutoff
    would be a disagreement.  Measured on one H100 80GB HBM3: the device exp returns subnormals down to an argument of
    745.0 and 0 from there on (correct rounding would give 2^-1074 up to 745.13); its last nonzero entries sit at r2 =
    1490.0 (ExpSquared, cutoff 1490.4), 185000 (Matern32, 185200), 111005 (Matern52, 111100) and 555025 (Exp, 555400)."""
    cls = PROFILES[prof][0]
    r2 = _sweep_r2(prof)
    x1 = np.sqrt(r2)[:, None]
    spec_k = _const(LOG_C, 1, None) * cls(metric=1.0)
    twin = _const(LOG_C, 2, [0]) * cls(metric=1.0, ndim=2, axes=[0]) * _const(0.0, 2, [0])
    assert spec_paths(spec_k)[0] == PROFILES[prof][1] and spec_paths(twin)[0] == 0
    # one-hot: a single x2 point with v = 1, and three x2 points with a one-hot v
    x2 = np.array([[0.0], [3.0], [-5.0]])
    for xx2, v in ((x2[:1], np.ones(1)), (x2, np.array([1.0, 0.0, 0.0]))):
        a = spec_k.matvec(x1, xx2, v)
        b = twin.matvec(_embed(x1), _embed(xx2), v)
        assert_bits_equal(a, b, prof)
    r2_dev = x1[:, 0] * x1[:, 0]
    past = r2_dev > CUTOFF[prof]
    record_property("interpreter_nonzero_past_cutoff", int(np.count_nonzero(b[past])))
    record_property("interpreter_subnormal_entries", int(np.count_nonzero((b != 0) & (np.abs(b) < 2.2250738585072014e-308))))
    record_property("last_nonzero_r2", float(r2_dev[b != 0].max()) if np.any(b != 0) else 0.0)
    assert np.all(a[past] == 0.0)


# ---- HODLR: the ACA, the leaves -------------------------------------------------------------------------------------

HODLR_FORMS = [f for f in SPECIALISED if f.nd == 1 and (f.name.endswith("_1d_iso_cS") or f in TWO_TERM)
               and not f.name.endswith(("c2E+cS", "Ec2+Sc", "S+E", "_S*E"))]


def _hodlr_run(kern, x, yerr, y, **kw):
    from george_b200.solvers._hodlr import HODLRSolver
    s = HODLRSolver()
    s.compute(kern, x, yerr, seed=42, **kw)
    nodes = s.nodes()
    piv, fac = [], []
    for i, nd in enumerate(nodes):
        if not nd["is_leaf"]:
            piv.append(s.pivots(i, nd["rank"]))
            if nd["rank"] > 0:
                fac.append(np.vstack(s.factors(i)))
    return {"nodes": nodes, "pivots": piv, "factors": fac, "logdet": s.log_determinant, "dot_solve": s.dot_solve(y),
            "solve": s.apply_inverse(y)[:, 0]}


@pytest.fixture
def no_cull(monkeypatch):
    for var in ("BGP_NO_GRAPH", "BGP_EVAL_MINB", "BGP_SMALL_RANK_LIMIT", "BGP_LEAF_COLS", "BGP_LEAF_FACTOR"):
        monkeypatch.delenv(var, raising=False)
    monkeypatch.setenv("BGP_NO_CULL", "1")  # the twin has no bound to cull with; culling's exactness is tested apart
    return monkeypatch


@pytest.mark.gpu
@pytest.mark.parametrize("rng_mode", ["pernode", "reference"])
@pytest.mark.parametrize("exhaust", ["lowrank", "dense"])
@pytest.mark.parametrize("tol", [1e-10, 1e-12])
@pytest.mark.parametrize("form", HODLR_FORMS, ids=repr)
def test_hodlr_matches_the_interpreter(gpu, no_cull, form, tol, exhaust, rng_mode):
    """The tree, ranks, draws, dense fallbacks, every pivot and every ACA factor bit for bit; the log-determinant and the
    solves within the up-sweep's atomics noise (as the culled scan against the exhaustive one)."""
    rng = np.random.default_rng(5)
    n = 3000
    x = np.sort(2.45e3 + rng.uniform(0.0, 300.0, n))[:, None]
    yerr = 0.2 * np.ones(n)
    y = np.sin(x[:, 0])
    kw = dict(min_size=100, tol=tol, rng_mode=rng_mode, exhaust=exhaust)
    a = _hodlr_run(form.kernel(), x, yerr, y, **kw)
    b = _hodlr_run(form.twin(), _embed(x), yerr, y, **kw)
    assert a["nodes"] == b["nodes"]
    assert sum(nd["rank"] for nd in a["nodes"]) > 0
    for (ra, ca), (rb, cb) in zip(a["pivots"], b["pivots"]):
        assert np.array_equal(ra, rb) and np.array_equal(ca, cb)
    assert len(a["factors"]) == len(b["factors"])
    for fa, fb in zip(a["factors"], b["factors"]):
        assert_bits_equal(fa, fb, "ACA factors")
    assert abs(a["logdet"] - b["logdet"]) <= 1e-13 * abs(b["logdet"])
    assert abs(a["dot_solve"] - b["dot_solve"]) <= 1e-12 * abs(b["dot_solve"])
    assert np.max(np.abs(a["solve"] - b["solve"])) <= 1e-12 * np.max(np.abs(b["solve"]))


@pytest.mark.gpu
@pytest.mark.parametrize("form", HODLR_FORMS, ids=repr)
def test_hodlr_leaf_factor_matches_the_interpreter(gpu, no_cull, form):
    """A tree whose root is its only leaf: the leaf factorisation alone, so the log-determinant and the solve are
    functions of the leaf factor and must agree bit for bit."""
    rng = np.random.default_rng(6)
    n = 700
    x = np.sort(2.45e3 + rng.uniform(0.0, 70.0, n))[:, None]
    yerr = 0.2 * np.ones(n)
    y = rng.normal(size=(n, 3))
    out = []
    for kern, xx in _routes(form, x)[:2]:
        from george_b200.solvers._hodlr import HODLRSolver
        s = HODLRSolver()
        s.compute(kern, xx, yerr, min_size=n, tol=1e-12, seed=42)
        assert len(s.nodes()) == 1
        out.append((s.log_determinant, s.apply_inverse(y)))
    assert_bits_equal(out[0][0], out[1][0], "leaf log-determinant")
    assert_bits_equal(out[0][1], out[1][1], "leaf solve")


# ---- the x1-gradient contraction of GP.grad_predict -------------------------------------------------------------------

def _grad_reference(prof, c, m, t, s):
    """d/dt of c f(m (t - s)^2) in extended precision from the float64 inputs; the Exp kernel's coincident-pair guard
    (float64 r2 below 2^-52 gives 0) applied as the kernels apply it"""
    import mpmath as mp
    mp.mp.prec = 160
    out = np.empty(len(t))
    arg = np.empty(len(t))
    for k, (ti, si) in enumerate(zip(t, s)):
        d64 = ti - si
        d = mp.mpf(ti) - mp.mpf(si)
        r2 = mp.mpf(m) * d * d
        if prof == "expsq":
            fp, a = -mp.mpf(0.5) * mp.exp(-r2 / 2), r2 / 2
        elif prof == "m32":
            r = mp.sqrt(3 * r2)
            fp, a = -mp.mpf(1.5) * mp.exp(-r), r
        elif prof == "m52":
            r = mp.sqrt(5 * r2)
            fp, a = -mp.mpf(5) / 6 * (1 + r) * mp.exp(-r), r
        else:
            r = mp.sqrt(r2)
            if d64 * d64 * m < 2.220446049250313e-16:
                fp, a = mp.mpf(0), r
            else:
                fp, a = -mp.exp(-r) / (2 * r), r
        out[k] = float(mp.mpf(c) * fp * 2 * mp.mpf(m) * d)
        arg[k] = float(a)
    return out, arg


def _c_and_m(form):
    """the float64 constant and inverse metric the device sees (exp on the host, as build_dev_program does)"""
    from george_b200._spec import OP_KERNEL, flatten
    spec = flatten(form.kernel())
    c, m = 1.0, None
    for i in range(spec.n_nodes):
        nd = spec.nodes[i]
        if nd.op == OP_KERNEL and nd.kernel_type == 8:  # BGP_K_CONSTANT
            c = math.exp(nd.params[0])
        elif nd.op == OP_KERNEL:
            m = math.exp(-nd.metric[0])
    return c, m


@pytest.mark.gpu
@pytest.mark.parametrize("form", ONE_TERM_1D, ids=repr)
def test_x1_gradient_contraction_within_ulps_of_mpmath(gpu, record_property, form):
    """kernel.x1_gradient_matvec (ScaledProfileGrad1D) and its twin (the interpreter's exact derivative): single
    entries through one-hot columns, within 4 ulp of the reference scaled by 1 + the exponent's argument; random
    contractions within eps * sum_j |term_j| (2 + argument_j).  Measured on one H100 80GB HBM3: at most 1.61 of the
    4 ulp, and at most 0.13 of the contraction bound.  A bare profile multiplies in the
    same order on both routes and must agree exactly."""
    import mpmath as mp
    prof = form.name.split("_")[0]
    c, m = _c_and_m(form)
    rng = np.random.default_rng(3)
    # single pairs: moderate distances, coincident pairs, and for Exp r2 across the 2^-52 gradient guard
    n = 256
    s = rng.uniform(-3.0, 3.0, n)
    d = rng.uniform(-4.0, 4.0, n)
    d[:8] = 0.0
    if prof == "exp":
        g = 2.220446049250313e-16
        d[8:120] = np.sqrt(np.linspace(g * (1 - 1e-3), g * (1 + 1e-3), 112) / m) * np.where(np.arange(112) % 2, 1, -1)
    t = s + d
    ref, arg = _grad_reference(prof, c, m, t, s)
    V = np.eye(n)
    worst = 0.0
    got = []
    for kern, emb in _routes(form, t[:, None])[:2]:
        x2 = _embed(s[:, None]) if emb.shape[1] == 2 else s[:, None]
        gi = kern.kernel.x1_gradient_matvec(emb, x2, V)[:, 0]
        zero = ref == 0
        assert np.all(gi[zero] == 0)
        err = np.abs(gi - ref)[~zero] / (EPS * np.abs(ref[~zero]) * (1.0 + arg[~zero]))
        worst = max(worst, float(np.max(err)))
        got.append(gi)
    record_property("entry_ulps", worst)
    assert worst <= 4.0, worst
    if form.name.endswith("_S"):
        assert np.array_equal(got[0], got[1])
    # contractions: 16 test points against 200 points with random weights
    t2 = rng.uniform(-3.0, 3.0, 16)
    s2 = rng.uniform(-3.0, 3.0, 200)
    v = rng.normal(size=200)
    terms = np.empty((16, 200))
    args = np.empty((16, 200))
    for i in range(16):
        gref, a = _grad_reference(prof, c, m, np.full(200, t2[i]), s2)
        terms[i], args[i] = gref * v, a
    ref_sum = np.array([float(mp.fsum(mp.mpf(x) for x in row)) for row in terms])
    bound = EPS * np.sum(np.abs(terms) * (2.0 + args), axis=1)
    worst = 0.0
    for kern, emb in _routes(form, t2[:, None])[:2]:
        x2 = _embed(s2[:, None]) if emb.shape[1] == 2 else s2[:, None]
        gsum = kern.kernel.x1_gradient_matvec(emb, x2, v)[:, 0]
        worst = max(worst, float(np.max(np.abs(gsum - ref_sum) / bound)))
    record_property("sum_bound_fraction", worst)
    assert worst <= 1.0, worst
