# -*- coding: utf-8 -*-
"""The HODLR symmetric factor K~ = W W^T (csrc/hodlr_sym.cu) and GP.sample on it.

* Small N: W = apply_symmetric_factor(I) against K~ assembled in numpy from the leaf blocks (K + diag(yerr^2)) and the
  nodes' ACA factors (``factors``); W^T; the orthonormality of every node's bases.
* Scale (bench.py's workloads): the symmetric log-determinant against the solver's, and the whitening identity
  (W Z)^T K~^-1 (W Z) = Z^T Z through the existing solve — an oracle that needs no dense matrix.
* GP.sample's contract, tree edge cases, failures and one statistics check.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# Bars: the targets the factorisation is built for; the measured values are from one H100 80GB HBM3 (SXM, 700 W).
TOL_FACTOR = 1e-13   # max |W W^T - K~| / max |K~|                                   (measured 2.5e-14)
TOL_TRANS = 1e-13    # max |W^T(I) - W(I)^T| / max |W|                               (measured 4.2e-15)
TOL_ORTH = 1e-13     # max |Q^T Q - I| over the nodes                                 (measured 4.7e-15)
TOL_LOGDET = 1e-12   # |symmetric_log_determinant - log_determinant| / |log_determinant| (measured 2.2e-13, cfg5)
TOL_WHITEN = 1e-9    # max |Y^T K~^-1 Y - Z^T Z| / max |Z^T Z|                        (measured 6.2e-12, cfg5)


def _native(kernel, x, yerr, **kw):
    from george_b200.solvers._hodlr import HODLRSolver
    s = HODLRSolver()
    x = np.asarray(x, dtype=np.float64)
    if x.ndim == 1:
        x = x[:, None]
    s.compute(kernel, x, yerr, **kw)
    return s, x


def _assemble(s, kernel, x, yerr):
    """K~ in numpy: exact leaf blocks, off-diagonal blocks Ur Vl^T of every internal node."""
    n = x.shape[0]
    K = kernel.get_value(x) + np.diag(np.asarray(yerr) ** 2)
    Kt = np.zeros((n, n))
    for i, nd in enumerate(s.nodes()):
        a, m, h = nd["start"], nd["size"], nd["half"]
        if nd["is_leaf"]:
            Kt[a:a + m, a:a + m] = K[a:a + m, a:a + m]
        else:
            Vl, Ur = s.factors(i)
            B = Ur @ Vl.T
            Kt[a + h:a + m, a:a + h] = B
            Kt[a:a + h, a + h:a + m] = B.T
    return Kt


def _kernels():
    from george_b200 import kernels as K
    return {
        "m32": (1.0 * K.Matern32Kernel(1.0), 1),
        "expsq": (1.0 * K.ExpSquaredKernel(1.0), 1),
        "quasiperiodic": (1.0 * K.ExpSquaredKernel(1.0) + 0.5 * K.ExpSine2Kernel(gamma=1.0, log_period=np.log(3.0)), 1),
        "general2d": (1.0 * K.ExpSquaredKernel([[4.0, 0.6], [0.6, 2.0]], ndim=2), 2),
    }


def _points(n, ndim, seed=3):
    rng = np.random.default_rng(seed)
    if ndim == 1:
        return np.sort(rng.uniform(0, 10 * n / 1000, n))
    x = rng.uniform(0, 4, (n, 2))
    return x[np.argsort(x[:, 0])]


# ---- 1. the factor at small N -------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["m32", "expsq", "quasiperiodic", "general2d"])
@pytest.mark.parametrize("n", [1000, 4096, 1537])
def test_factor_identity(gpu, record_property, name, n):
    kernel, ndim = _kernels()[name]
    x = _points(n, ndim)
    yerr = 0.1 + 0.05 * np.random.default_rng(1).uniform(size=n)
    s, x = _native(kernel, x, yerr, min_size=64, tol=1e-12, exhaust="lowrank")
    Kt = _assemble(s, kernel, x, yerr)
    W = s.apply_symmetric_factor(np.eye(n))
    err = np.max(np.abs(W @ W.T - Kt)) / np.max(np.abs(Kt))
    Wt = s.apply_symmetric_factor(np.eye(n), transpose=True)
    terr = np.max(np.abs(Wt - W.T)) / np.max(np.abs(W))
    orth = s.symmetric_factor_orthogonality()
    record_property("factor_err", err)
    record_property("transpose_err", terr)
    record_property("orth_err", orth)
    assert err <= TOL_FACTOR and terr <= TOL_TRANS and orth <= TOL_ORTH
    # log|K~| three ways: the symmetric factor, the solver, numpy
    ld = np.linalg.slogdet(Kt)[1]
    assert abs(s.symmetric_log_determinant - s.log_determinant) <= TOL_LOGDET * abs(s.log_determinant)
    assert abs(s.symmetric_log_determinant - ld) <= 1e-10 * abs(ld)
    # a vector and a matrix give the same columns
    z = np.random.default_rng(2).standard_normal(n)
    assert np.allclose(s.apply_symmetric_factor(z), W @ z, rtol=0, atol=1e-12 * np.max(np.abs(W)) * np.sqrt(n))


# ---- 2./3. log-determinant and whitening at scale ------------------------------------------------------------------

@pytest.mark.parametrize("case", [("cfg3", 65536, 256), ("cfg3", 262144, 256), ("cfg2", 65536, 100),
                                  ("cfg5", 131072, 100)])
def test_logdet_and_whitening_at_scale(gpu, record_property, case):
    name, n, min_size = case
    from george_b200 import kernels as K
    kernel = {"cfg3": 1.0 * K.Matern32Kernel(1.0), "cfg2": 1.0 * K.ExpSquaredKernel(1.0),
              "cfg5": 1.0 * K.ExpSquaredKernel(1.0) + 0.5 * K.ExpSine2Kernel(gamma=1.0, log_period=np.log(3.0))}[name]
    rng = np.random.default_rng(1234)
    x = np.sort(rng.uniform(0, 10 * n / 1000, n))
    s, x = _native(kernel, x, 0.1 * np.ones(n), min_size=min_size, tol=1e-10, seed=42, exhaust="lowrank")
    ld, sld = s.log_determinant, s.symmetric_log_determinant
    rel = abs(sld - ld) / abs(ld)
    record_property("logdet_rel", rel)
    assert rel <= TOL_LOGDET
    Z = np.random.default_rng(7).standard_normal((n, 8))
    Y = s.apply_symmetric_factor(Z)
    G = Y.T @ s.apply_inverse(Y)
    werr = np.max(np.abs(G - Z.T @ Z)) / np.max(np.abs(Z.T @ Z))
    record_property("whiten_err", werr)
    assert werr <= TOL_WHITEN
    # deterministic: the same factorisation applies with the same bits
    assert np.array_equal(s.apply_symmetric_factor(Z[:, :1]), Y[:, :1])


# ---- 4. GP.sample --------------------------------------------------------------------------------------------------

def _gp(n=2000, seed=0, ell=1.0, **kw):
    import george_b200 as george
    from george_b200 import kernels
    t = np.sort(np.random.default_rng(seed).uniform(0, 10, n))
    gp = george.GP(1.0 * kernels.Matern32Kernel(ell), mean=0.7, solver=george.HODLRSolver,
                   **dict(dict(min_size=64, tol=1e-10, exhaust="lowrank"), **kw))
    gp.compute(t, 0.1)
    return gp, t


def test_gp_sample_contract(gpu):
    gp, t = _gp()
    n = len(t)
    g = np.random.default_rng(11)
    ref = np.random.default_rng(11)
    z = ref.standard_normal((5, n))
    vec, solver, alpha, computed = gp.get_parameter_vector(), gp.solver, getattr(gp, "_alpha", None), gp.computed
    d = gp.sample(size=5, rng=g)
    assert np.array_equal(d, gp.solver.sample_prior(z) + gp._call_mean(gp._x))
    assert np.array_equal(g.standard_normal(3), ref.standard_normal(3))  # advanced by exactly one (5, N) draw
    assert np.array_equal(gp.get_parameter_vector(), vec) and gp.solver is solver and gp.computed == computed
    assert getattr(gp, "_alpha", None) is alpha
    assert np.array_equal(gp.sample(size=5, rng=np.random.default_rng(11)), d)  # same seed, same bits
    one = gp.sample(size=1, rng=np.random.default_rng(3))
    assert one.shape == (n,)
    assert gp.sample(size=0, rng=np.random.default_rng(3)).shape == (0, n)
    many = gp.sample(size=130, rng=np.random.default_rng(4))  # 64 + 64 + 2 columns
    z = np.random.default_rng(4).standard_normal((130, n))
    W = gp.solver.solver.apply_symmetric_factor(np.eye(n))
    assert np.allclose(many, z @ W.T + 0.7, rtol=0, atol=1e-11)
    assert np.array_equal(many[:64], gp.sample(size=64, rng=np.random.default_rng(4)))
    with pytest.raises(NotImplementedError):  # rng=None keeps the reference's route
        gp.sample()


def test_reused_handle_never_serves_a_stale_factor(gpu):
    import george_b200 as george
    from george_b200.solvers._hodlr import HODLRSolver as Native
    gp, t = _gp()
    gp.sample(size=2, rng=np.random.default_rng(0))
    gp.set_parameter_vector(gp.get_parameter_vector() + 0.3)
    gp.compute(t, 0.1)  # picks up a parked handle that holds theta_1's factor
    got = gp.sample(size=2, rng=np.random.default_rng(5))
    Native.release_parked()
    fresh, _ = _gp()
    fresh.set_parameter_vector(gp.get_parameter_vector())
    fresh.compute(t, 0.1)
    assert np.array_equal(got, fresh.sample(size=2, rng=np.random.default_rng(5)))
    assert isinstance(gp.solver, george.HODLRSolver)


# ---- 5. tree edge cases --------------------------------------------------------------------------------------------

def test_root_leaf(gpu):
    from george_b200 import kernels
    n = 100  # < 2 min_size: the root is one leaf, W = L D^1/2
    x = np.sort(np.random.default_rng(0).uniform(0, 5, n))
    kernel = 1.0 * kernels.ExpSquaredKernel(1.0)
    s, x = _native(kernel, x, 0.1 * np.ones(n), min_size=64, tol=1e-12)
    K = kernel.get_value(x) + 0.01 * np.eye(n)
    W = s.apply_symmetric_factor(np.eye(n))
    assert np.allclose(np.triu(W, 1), 0.0)
    assert np.max(np.abs(W @ W.T - K)) <= TOL_FACTOR * np.max(np.abs(K))
    assert abs(s.symmetric_log_determinant - np.linalg.slogdet(K)[1]) <= 1e-12 * n


@pytest.mark.parametrize("n", [1000, 777])
def test_rank_zero_nodes_and_unequal_halves(gpu, n):
    from george_b200 import kernels
    # two clusters far apart: the blocks between them are exactly zero, so with exhaust="lowrank" those nodes have rank 0
    rng = np.random.default_rng(1)
    x = np.sort(np.concatenate([rng.uniform(0, 1, n // 2), rng.uniform(1000, 1001, n - n // 2)]))
    kernel = 1.0 * kernels.ExpSquaredKernel(0.05)
    yerr = 0.1 * np.ones(n)
    s, x = _native(kernel, x, yerr, min_size=64, tol=1e-12, exhaust="lowrank")
    assert s.nodes()[0]["rank"] == 0
    Kt = _assemble(s, kernel, x, yerr)
    W = s.apply_symmetric_factor(np.eye(n))
    assert np.max(np.abs(W @ W.T - Kt)) <= TOL_FACTOR * np.max(np.abs(Kt))
    assert np.allclose(s.apply_symmetric_factor(np.eye(n), transpose=True), W.T, rtol=0, atol=TOL_TRANS)
    ld = np.linalg.slogdet(Kt)[1]
    assert abs(s.symmetric_log_determinant - ld) <= 1e-10 * abs(ld)


# ---- 6. failures ---------------------------------------------------------------------------------------------------

def test_indefinite_hodlr_matrix_raises_and_gp_survives(gpu):
    import george_b200 as george
    from george_b200 import kernels
    # ExpSquared with little noise at tol = 0.1: the ACA's loose blocks make K~ indefinite; the first seed whose
    # assembled K~ has a clearly negative eigenvalue is used (the loop must find one)
    for seed in range(8):
        rng = np.random.default_rng(seed)
        n = 1000
        t = np.sort(rng.uniform(0, 10, n))
        y = np.sin(t)
        gp = george.GP(1.0 * kernels.ExpSquaredKernel(0.5), solver=george.HODLRSolver, min_size=50)
        gp.compute(t, 1e-3)
        Kt = _assemble(gp.solver.solver, gp.kernel, t[:, None], 1e-3 * np.ones(n))
        ev = np.linalg.eigvalsh(Kt)
        if ev[0] < -1e-8 * ev[-1]:
            break
    else:
        pytest.fail("no seed gave an indefinite HODLR matrix")
    ll, mu = gp.log_likelihood(y), gp.predict(y, t[:50], return_cov=False)
    with pytest.raises(np.linalg.LinAlgError, match="not positive definite: node"):
        gp.sample(size=3, rng=np.random.default_rng(0))
    assert np.array_equal(gp.log_likelihood(y), ll)
    assert np.array_equal(gp.predict(y, t[:50], return_cov=False), mu)


def test_negative_leaf_pivot_raises(gpu):
    from george_b200 import kernels
    # No kernel shipped here is indefinite, and yerr^2 >= 0, so a negative pivot comes from round-off: a noise-free,
    # numerically rank-one leaf (a length scale 1e4 times the data's span) runs its L D L^T pivots down to the rounding
    # level, where they take either sign or vanish.  compute() accepts that leaf (log|D|); the symmetric factor does not.
    n = 200
    x = np.linspace(0, 1, n)
    s, x = _native(1.0 * kernels.ExpSquaredKernel(1e8), x, np.zeros(n), min_size=64, tol=1e-12)
    with pytest.raises(np.linalg.LinAlgError, match="leaf"):
        s.symmetric_log_determinant


@pytest.mark.parametrize("n", [1000, 1537])
def test_dense_fallback_nodes(gpu, record_property, n):
    from george_b200 import kernels
    # Matern32 at this spacing runs out of rows: with exhaust="dense" (the solver's default) the ACA returns the dense
    # block, whose columns are numerically dependent (condition ~1e20 after equilibration).  CholeskyQR cannot
    # orthonormalise them; the Householder path does, and W still reproduces K~.
    kernel = 1.0 * kernels.Matern32Kernel(1.0)
    yerr = 0.1 * np.ones(n)
    s, x = _native(kernel, _points(n, 1), yerr, min_size=64, tol=1e-12)
    assert any(d["dense_fallback"] for d in s.nodes() if not d["is_leaf"])
    Kt = _assemble(s, kernel, x, yerr)
    W = s.apply_symmetric_factor(np.eye(n))
    err = np.max(np.abs(W @ W.T - Kt)) / np.max(np.abs(Kt))
    orth = s.symmetric_factor_orthogonality()
    record_property("factor_err", err)
    record_property("orth_err", orth)
    assert err <= TOL_FACTOR and orth <= TOL_ORTH
    ld = np.linalg.slogdet(Kt)[1]
    assert abs(s.symmetric_log_determinant - ld) <= 1e-10 * abs(ld)


def test_nan_inputs_raise(gpu):
    from george_b200 import kernels
    n = 500
    x = np.sort(np.random.default_rng(0).uniform(0, 5, n))
    x[123] = np.nan
    s, x = _native(1.0 * kernels.Matern32Kernel(1.0), x, 0.1 * np.ones(n), min_size=64, tol=1e-10, exhaust="lowrank")
    with pytest.raises(np.linalg.LinAlgError, match="leaf"):
        s.apply_symmetric_factor(np.ones(n))
    # the device is still usable
    s2, _ = _native(1.0 * kernels.Matern32Kernel(1.0), np.linspace(0, 5, n), 0.1 * np.ones(n), min_size=64, tol=1e-10,
                    exhaust="lowrank")
    assert np.isfinite(s2.symmetric_log_determinant)


def test_sharded_handles_are_rejected(gpu):
    import george_b200 as george
    from george_b200 import kernels
    from george_b200.solvers._hodlr import HODLRSolver
    n = 4096
    x = np.sort(np.random.default_rng(0).uniform(0, 40, n))[:, None]
    s = HODLRSolver()
    s.compute(1.0 * kernels.Matern32Kernel(1.0), x, 0.1 * np.ones(n), min_size=64, tol=1e-10, shard_rank=0,
              shard_count=2)
    with pytest.raises(ValueError, match="sharded"):
        s.apply_symmetric_factor(np.ones(n))
    with pytest.raises(ValueError, match="sharded"):
        s.symmetric_log_determinant
    # the GP route: ShardedHODLRSolver has no sample_prior hook, so GP.sample stays apply_sqrt's NotImplementedError
    from george_b200.parallel import ShardedHODLRSolver
    assert getattr(ShardedHODLRSolver, "sample_prior", None) is None


# ---- 7. statistics -------------------------------------------------------------------------------------------------

def test_sample_covariance(gpu):
    gp, t = _gp(n=2048, ell=0.5)
    size = 20000
    d = gp.sample(size=size, rng=np.random.default_rng(9)) - 0.7
    Kt = _assemble(gp.solver.solver, gp.kernel, t[:, None], 0.1 * np.ones(len(t)))
    S = d.T @ d / size  # the mean is known
    sigma = np.sqrt((Kt ** 2 + np.outer(np.diag(Kt), np.diag(Kt))) / size)  # std of a Wishart entry / size
    assert np.all(np.abs(S - Kt) <= 6 * sigma)
