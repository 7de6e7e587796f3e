# -*- coding: utf-8 -*-
"""The device paths on non-finite and degenerate inputs.

* Evaluators: kernel values, hyper-gradients and x-gradients at NaN / +-inf coordinates, pairs 1e200 apart (r2 = +inf),
  duplicated points and overflowing parameters, against the reference's own values in tests/golden/reference_nonfinite.npz
  (make_golden_nonfinite.py): the NaN pattern must be identical and the finite entries agree to the usual tolerances.
* ACA decisions: a NaN row at the root's first draw, at a later draw behind a sub-threshold row, and a NaN column in a
  group that bound culling would otherwise skip.  Every node's rank, pivots, words drawn and exhaustion flag equal the
  oracle's under the one NaN rule (DESIGN.md §2), on every evaluation route, in both RNG and both exhaustion modes.
* End to end: the dense path's outcome under quiet=False and quiet=True is the reference's (value, -inf or exception
  class, never a device error); HODLR gives -inf exactly where the oracle's likelihood is not finite.  Gradient,
  prediction, then the same GP and parked HODLR handle on a well-posed problem.  A singular Woodbury matrix above the
  small-LU size.  Batch members with an overflowing parameter are -inf and leave their neighbours bit for bit equal to
  the one-at-a-time path; batch_predict raises the member's factorisation error, as predict does.
N stays small: a NaN pivot drives a node to full rank (in the reference too).
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import aca_draw_model as M

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_nonfinite as G  # noqa: E402  (the same problem definitions the golden file was made from)

pytestmark = pytest.mark.gpu

GOLD = np.load(os.path.join(HERE, "golden", "reference_nonfinite.npz"))
KERNELS = [str(k) for k in GOLD["manifest__kernels"]]
E2E = [str(c) for c in GOLD["manifest__e2e"]]
LL_RTOL = 1e-9        # dense against the reference
HODLR_LL_RTOL = 1e-7  # against the oracle: measured 6.3e-9 at log_M = +720 (K = 1.5 everywhere, cond ~ 1e4), H100


def _kernel(name):
    from george_b200 import kernels
    return G.make_kernel(G.kernel_zoo(kernels), name)


def _same(got, ref, rtol, atol, what):
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert np.array_equal(np.isnan(got), np.isnan(ref)), (what, np.argwhere(np.isnan(got) != np.isnan(ref))[:8])
    fin = np.isfinite(ref)
    assert np.array_equal(np.isfinite(got), fin), (what, np.argwhere(np.isfinite(got) != fin)[:8])
    assert np.array_equal(got[np.isinf(ref)], ref[np.isinf(ref)]), what
    np.testing.assert_allclose(got[fin], ref[fin], rtol=rtol, atol=atol, err_msg=what)


def check_evaluators(name):
    k, nd = _kernel(name)
    np.testing.assert_array_equal(k.get_parameter_vector(include_frozen=True), GOLD[name + "__params"])
    x1, x2 = G.inputs(nd)
    rtol = 5e-12 if "ratquad" in name else 1e-12
    _same(k.get_value(x1, x2), GOLD[name + "__value"], rtol, 1e-15, name + " value")
    _same(k.get_gradient(x1, x2, include_frozen=True), GOLD[name + "__grad"], rtol, 1e-14, name + " grad")
    _same(k.get_x1_gradient(x1, x2), GOLD[name + "__x1grad"], rtol, 1e-14, name + " x1grad")


@pytest.mark.parametrize("name", KERNELS)
def test_evaluators_match_reference(gpu, name):
    """Default build of the kernel matrix (kmat): ProfileND for one radial kernel in 1-3 dimensions, the interpreter
    for the rest.  The specialised 1-D evaluators of the matvec, leaves and ACA are checked at r2 = +inf by
    test_matvec_far_points_are_nan."""
    check_evaluators(name)


def test_generic_build_matches_reference(gpu):
    """BGP_KMAT_GENERIC (read once per process) routes every kernel matrix through the interpreter."""
    env = dict(os.environ, BGP_KMAT_GENERIC="1", PYTHONPATH=os.pathsep.join([os.path.dirname(HERE), HERE]))
    code = ("import test_gpu_nonfinite as T\nfor n in T.KERNELS: T.check_evaluators(n)\nprint('generic ok', len(T.KERNELS))")
    r = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=os.path.dirname(HERE), capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0 and "generic ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


@pytest.mark.parametrize("kname", ["m32", "m52"])
def test_matvec_far_points_are_nan(gpu, kname):
    """The shape-dispatched matvec (the predictive mean): a test point 1e200 away has r2 = +inf, where the Matern
    forms are (1 + inf) exp(-inf) = NaN in the reference; nearby test points are unaffected."""
    import george_b200 as george
    from george_b200 import kernels
    k = 2.0 * (kernels.Matern32Kernel(0.7) if kname == "m32" else kernels.Matern52Kernel(0.7))
    rng = np.random.default_rng(3)
    x = np.sort(rng.uniform(0, 10, 300))
    y = np.sin(x)
    gp = george.GP(k)
    gp.compute(x, 0.1)
    t = np.array([0.5, 1e200, 3.0, -1e200, np.inf])
    mu = gp.predict(y, t, return_cov=False)
    assert np.array_equal(np.isnan(mu), [False, True, False, True, True]), mu
    alpha = np.linalg.solve(k.get_value(x[:, None]) + 0.01 * np.eye(len(x)), y)
    np.testing.assert_allclose(mu[[0, 2]], k.get_value(t[[0, 2], None], x[:, None]) @ alpha, rtol=1e-9)


# ---- ACA decisions on NaN rows ---------------------------------------------------------------------------------------
ACA = dict(n=1031, min_size=60, seed=42)


@pytest.fixture
def clean_env(monkeypatch):
    for var in ("BGP_NO_GRAPH", "BGP_NO_CULL", "BGP_EVAL_MINB"):
        monkeypatch.delenv(var, raising=False)
    return monkeypatch


def _nan_problem(where, chained):
    P = M.Problem(chained=chained, **ACA)
    d = P.draws(0)
    nd = P.nodes[0]
    if where == "first_row":
        P.place(0, 3, 0.5, d)
        nan_at = nd["start"] + nd["half"] + int(d.rows[0])
    elif where == "later_row":
        P.place(0, 1, 0.5, d)
        P.place(0, 4, M.SUB_THRESHOLD, d)   # rejected just before: its arg-max column must not be reused
        nan_at = nd["start"] + nd["half"] + int(d.rows[5])
    elif where == "culled_column":
        # the moved partner of a special row stretches the node's column box into the rows; draw 0 must stay outside
        # it, so that the node-level cull (not only the 128-column group's) sees the NaN column
        c = min(range(1, 9), key=lambda q: int(d.rows[q]))
        assert int(d.rows[c]) < int(d.rows[0])
        P.place(0, c, 0.5, d)
        col = P.pairs[0][0][1]
        nan_at = nd["start"] + (0 if col // 128 != 0 else 300)   # a 128-column group far from every row
    else:
        raise ValueError(where)
    x = P.x
    x[nan_at, 0] = np.nan
    return P, x


_ORACLE = {}


def _oracle_nodes(oracle, where, rng_mode, exhaust):
    key = (where, rng_mode, exhaust)
    if key not in _ORACLE:
        from george_b200._spec import flatten
        P, x = _nan_problem(where, rng_mode == "reference")
        h = oracle.HODLR(flatten(P.kernel()), x, 0.1 * np.ones(P.n), min_size=P.min_size, tol=P.tol, seed=P.seed,
                         rng_mode=1 if rng_mode == "reference" else 0, exhaust=1 if exhaust == "lowrank" else 0)
        nodes = h.nodes()
        piv = [h.pivots(i, nd["rank"]) if not nd["is_leaf"] else None for i, nd in enumerate(nodes)]
        _ORACLE[key] = (nodes, piv)
    return _ORACLE[key]


# rng_mode = "reference" always runs aca_kernel (one CTA per node, no culling, no graph): one route covers it
ROUTES = [("pernode", "default"), ("pernode", "no_cull"), ("pernode", "no_graph"), ("reference", "default")]


@pytest.mark.parametrize("rng_mode,route", ROUTES)
@pytest.mark.parametrize("exhaust", ["lowrank", "dense"])
@pytest.mark.parametrize("where", ["first_row", "later_row", "culled_column"])
def test_nan_aca_decisions(gpu, oracle, clean_env, where, rng_mode, exhaust, route):
    from george_b200.solvers._hodlr import HODLRSolver
    if route == "no_cull":
        clean_env.setenv("BGP_NO_CULL", "1")
    if route == "no_graph":
        clean_env.setenv("BGP_NO_GRAPH", "1")
    P, x = _nan_problem(where, rng_mode == "reference")
    s = HODLRSolver()
    s.compute(P.kernel(), x, 0.1 * np.ones(P.n), min_size=P.min_size, tol=P.tol, seed=P.seed, rng_mode=rng_mode,
              exhaust=exhaust, rank_capacity=0)
    onodes, opiv = _oracle_nodes(oracle, where, rng_mode, exhaust)
    nodes = s.nodes()
    assert len(nodes) == len(onodes)
    full = 0
    for i, (nd, od) in enumerate(zip(nodes, onodes)):
        assert (nd["start"], nd["size"], bool(nd["is_leaf"])) == (od["start"], od["size"], bool(od["is_leaf"]))
        if nd["is_leaf"]:
            continue
        got = (nd["rank"], nd["rng_draws"], nd["dense_fallback"])
        assert got == (od["rank"], od["rng_draws"], od["dense_fallback"]), (i, got, od)
        if not (exhaust == "dense" and od["dense_fallback"]):
            rows, cols = s.pivots(i, nd["rank"])
            assert list(rows) == list(opiv[i][0]) and list(cols) == list(opiv[i][1]), i
        full += nd["rank"] >= 64   # a NaN drives the node to (near) full rank; steered nodes stop at 3
    assert full >= 2 and not np.isfinite(s.log_determinant)
    del s


# ---- end to end ------------------------------------------------------------------------------------------------------
def _gp(solver, vec=None):
    import george_b200 as george
    from george_b200 import kernels
    k = G.e2e_kernel(kernels, vec)
    if solver == "basic":
        return george.GP(k)
    tol = 0.1 if solver == "hodlr_default" else 1e-10
    return george.GP(k, solver=george.HODLRSolver, tol=tol, min_size=8, seed=42)


def _oracle_ll(oracle, x, yerr, y, vec, tol):
    from george_b200 import kernels
    from george_b200._spec import flatten
    import george_b200 as george
    sigma = np.sqrt(yerr ** 2 + george.gp.TINY)
    with np.errstate(all="ignore"):
        o = oracle.HODLR(flatten(G.e2e_kernel(kernels, vec)), x, sigma, min_size=8, tol=tol, seed=42,
                         rng_mode=1 if tol > 1e-6 else 0)
        ll = -0.5 * (len(x) * np.log(2 * np.pi) + o.log_determinant) - 0.5 * o.dot_solve(y)
    return ll if np.isfinite(ll) else -np.inf


def _recover(gp, solver, oracle, record_property):
    """The same GP (and, for HODLR, the parked native handle the failed compute left) on the clean problem."""
    from george_b200 import _lib, kernels
    x, yerr, y, _, _ = G.e2e_problem("clean")
    gp.set_parameter_vector(G.e2e_kernel(kernels, None).get_parameter_vector())
    gp.compute(x, yerr)
    ll = gp.log_likelihood(y)
    if solver == "basic":
        ref, tol = float(GOLD["e2e__clean__ll"]), 1e-12
    else:
        ref, tol = _oracle_ll(oracle, x, yerr, y, None, 0.1 if solver == "hodlr_default" else 1e-10), LL_RTOL
    record_property("recovery_rel_err", abs(ll - ref) / abs(ref))
    assert abs(ll - ref) <= tol * abs(ref), (ll, ref)
    assert _lib.load().bgp_dev_synchronize() == 0


def _outcome(fn):
    """"finite", "-inf" or the class name of the exception ``fn`` raises (a device error fails the test)."""
    from george_b200._lib import BGPError
    try:
        v = fn()
    except BGPError:
        raise
    except ValueError as exc:
        return type(exc).__name__
    return "finite" if np.isfinite(v) else ("-inf" if v == -np.inf else repr(v))


def _is_error(outcome):
    return outcome.isidentifier() and outcome != "finite"   # an exception class name, not "-inf" or a number


def _raises_like(got, ref):
    """A ValueError subclass wherever the reference raises one (LinAlgError is one)."""
    from numpy.linalg import LinAlgError
    classes = {"ValueError": ValueError, "LinAlgError": LinAlgError}
    return got in classes and issubclass(classes[got], classes[ref])


@pytest.mark.parametrize("solver", ["basic", "hodlr_default", "hodlr_tight"])
@pytest.mark.parametrize("case", E2E)
def test_end_to_end_outcome_and_recovery(gpu, oracle, record_property, case, solver):
    """Dense: the outcome of ``log_likelihood`` under quiet=False and quiet=True is the reference's (its value, -inf
    or the exception class).  HODLR: -inf where the oracle's log-likelihood is not finite (the HODLR solver, like the
    reference's, raises nothing on a NaN), its value where it is.  Then gradient, prediction and recovery."""
    import george_b200 as george
    x, yerr, y, _, vec = G.e2e_problem(case)
    tol = 0.1 if solver == "hodlr_default" else 1e-10

    def ll(quiet):
        gp = _gp(solver, vec)
        if not quiet:
            gp.compute(x, yerr)
        else:
            try:
                gp.compute(x, yerr)
            except ValueError:
                pass
        return gp.log_likelihood(y, quiet=quiet)

    loud, silent = _outcome(lambda: ll(False)), _outcome(lambda: ll(True))
    record_property("outcome", (loud, silent))
    if solver == "basic":
        ref_loud, ref_quiet = str(GOLD["e2e__%s__outcome" % case]), str(GOLD["e2e__%s__quiet" % case])
        ref_quiet = ref_quiet if _is_error(ref_quiet) else ("finite" if np.isfinite(float(ref_quiet)) else "-inf")
        for got, ref in ((loud, ref_loud), (silent, ref_quiet)):
            assert (_raises_like(got, ref) if _is_error(ref) else got == ref), (got, ref)
        expect_finite = ref_loud == "finite"
        ref_ll = float(GOLD["e2e__%s__ll" % case]) if expect_finite else None
    else:
        ref_ll = _oracle_ll(oracle, x, yerr, y, vec, tol)
        expect_finite = bool(np.isfinite(ref_ll))
        assert loud == silent == ("finite" if expect_finite else "-inf"), (loud, silent, ref_ll)

    gp = _gp(solver, vec)
    try:
        gp.compute(x, yerr)
    except ValueError:
        assert not expect_finite
    if expect_finite and case != "dup_yerr0":   # cond(K) ~ 1e16 at yerr = 0: only the outcome class is stable
        v = gp.log_likelihood(y)
        assert abs(v - ref_ll) <= (LL_RTOL if solver == "basic" else HODLR_LL_RTOL) * abs(ref_ll), (v, ref_ll)

    # gradient: the reference's quiet zeros when the likelihood fails on the dense path; on HODLR (no exception) the
    # NaN reaches it; where the likelihood is finite, a central difference of the likelihood
    g = gp.grad_log_likelihood(y, quiet=True)
    if not expect_finite:
        if solver == "basic":
            assert np.array_equal(g, np.zeros(len(gp))), g
        else:
            assert np.array_equal(g, np.zeros(len(gp))) or not np.any(np.isfinite(g)), g
    elif case != "dup_yerr0" and solver == "basic":
        p0, h, fd = gp.get_parameter_vector(), 1e-5, np.empty(len(gp))
        for k in range(len(gp)):
            vals = []
            for sgn in (1, -1):
                p = p0.copy()
                p[k] += sgn * h
                gp.set_parameter_vector(p)
                vals.append(gp.log_likelihood(y))
            fd[k] = (vals[0] - vals[1]) / (2 * h)
        gp.set_parameter_vector(p0)
        np.testing.assert_allclose(g, fd, rtol=1e-5, atol=1e-5 * max(np.max(np.abs(fd)), 1e-300))
    elif case != "dup_yerr0" and solver == "hodlr_tight":
        # against the dense gradient: a difference quotient of the HODLR likelihood is not usable here (its 1e-8
        # relative error at log_M = +720 moves with the parameters)
        gd = _gp("basic", vec)
        gd.compute(x, yerr)
        gref = gd.grad_log_likelihood(y)
        record_property("grad_rel_err", float(np.max(np.abs(g - gref) / np.maximum(np.abs(gref), 1e-300))))
        np.testing.assert_allclose(g, gref, rtol=1e-5, atol=1e-9 * np.max(np.abs(gref)))

    # prediction: the dense formula where the likelihood is finite; a ValueError or an all-NaN mean where it is not
    ts = np.linspace(0, 10, 7)
    if expect_finite:
        mu, var = gp.predict(y, ts, return_var=True)
        assert np.all(np.isfinite(mu)) and np.all(np.isfinite(var))
        if case != "dup_yerr0" and solver != "hodlr_default":
            k = gp.kernel
            K = k.get_value(x[:, None]) + np.diag(yerr ** 2 + george.gp.TINY)
            np.testing.assert_allclose(mu, k.get_value(ts[:, None], x[:, None]) @ np.linalg.solve(K, y), rtol=1e-6,
                                       atol=1e-9 * np.max(np.abs(y)))
    else:
        try:
            mu = gp.predict(y, ts, return_cov=False)
        except ValueError as exc:
            from george_b200._lib import BGPError
            assert not isinstance(exc, BGPError)
        else:
            assert np.all(np.isnan(mu)), mu
    _recover(gp, solver, oracle, record_property)


def test_singular_woodbury_matrix_above_the_small_path(gpu, oracle, record_property):
    """Two identical points, one in each half of the root, and no noise, as in test_gpu_hodlr.py's FullPivLU case but
    with r = 80: S is 160 x 160 and goes through the partial-pivoting blocked LU instead of the truncating small path.
    The outcome class (finite or not, log-det and solve) must be the oracle's; the solve difference is recorded."""
    from george_b200 import kernels as K
    from george_b200.solvers._hodlr import HODLRSolver
    from george_b200._spec import flatten
    rng = np.random.default_rng(8)
    n = 160
    x = np.sort(rng.uniform(0, 4, n))
    x[120] = x[40]
    x = x[:, None]
    yerr = np.zeros(n)
    y = np.sin(x[:, 0])
    kernel = 1.0 * K.ExpKernel(0.25)     # exactly rank 1 between sorted halves: the root stores its block densely
    s = HODLRSolver()
    s.compute(kernel, x, yerr, min_size=80, tol=1e-12, seed=42, rng_mode="reference")
    o = oracle.HODLR(flatten(kernel), x, yerr, min_size=80, tol=1e-12, seed=42, rng_mode=1)
    assert s.nodes()[0]["rank"] == 80 and o.nodes()[0]["rank"] == 80
    a, ao = s.apply_inverse(y)[:, 0], o.apply_inverse(y)
    ld, ldo = s.log_determinant, o.log_determinant
    record_property("logdet", (ld, ldo))
    scale = np.linalg.norm(ao)
    rel = float(np.linalg.norm(a - ao) / scale) if np.isfinite(scale) and scale > 0 else float("nan")
    record_property("solve_rel_diff", rel)
    record_property("solve_norms", (float(np.linalg.norm(a)), float(scale)))
    assert np.isfinite(ld) == np.isfinite(ldo)
    assert bool(np.all(np.isfinite(a))) == bool(np.all(np.isfinite(ao)))


# ---- batch paths -----------------------------------------------------------------------------------------------------
def test_batch_member_with_overflowing_parameter(gpu):
    import george_b200 as george
    from george_b200 import kernels
    x, yerr, y, _, _ = G.e2e_problem("clean")
    gp = george.GP(G.e2e_kernel(kernels, None))
    gp.compute(x, yerr)
    p0 = gp.get_parameter_vector()
    vecs = np.stack([p0, p0 + [800.0, 0.0], p0 + [0.0, -720.0] , p0 + [0.01, 0.02]])
    bad = [1, 2]
    llb = gp.batch_log_likelihood(vecs, y, quiet=True)
    llg, gb = gp.batch_grad_log_likelihood(vecs, y, quiet=True, return_log_likelihood=True)
    ts = np.linspace(0, 10, 9)
    for b in range(len(vecs)):
        gp.set_parameter_vector(vecs[b])
        ll1 = gp.log_likelihood(y, quiet=True)
        g1 = gp.grad_log_likelihood(y, quiet=True)
        if b in bad:
            assert llb[b] == -np.inf and llg[b] == -np.inf and ll1 == -np.inf
        else:
            assert llb[b] == ll1 and llg[b] == ll1
            assert np.array_equal(gb[b], g1)
    gp.set_parameter_vector(p0)
    good = [0, 3]
    mub, varb = gp.batch_predict(vecs[good], y, ts, return_var=True)
    # predict has no quiet mode: the loop raises the bad member's factorisation error (LinAlgError), and so does the batch
    from numpy.linalg import LinAlgError
    with pytest.raises(LinAlgError):
        gp.batch_predict(vecs, y, ts, return_var=True)
    gp.set_parameter_vector(vecs[1])
    with pytest.raises(LinAlgError):
        gp.predict(y, ts, return_var=True)
    for i, b in enumerate(good):
        gp.set_parameter_vector(vecs[b])
        mu1, var1 = gp.predict(y, ts, return_var=True)
        assert np.array_equal(mub[i], mu1) and np.array_equal(varb[i], var1)
