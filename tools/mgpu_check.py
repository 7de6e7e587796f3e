# -*- coding: utf-8 -*-
"""Multi-GPU parity probe (run under torchrun): sharded HODLR (sub-tree per rank + one all-gather) must reproduce the
single-GPU factorisation — same per-node RNG streams, so log-det / solve / gradient terms agree to rounding.  The
gradient leg runs the collective grad_terms (each rank streams K^-1 over its own columns; all-reduce of g, all-gather of
the diagonal) against the single-GPU grad_terms on rank 0.  The predict leg runs the collective predictive (each rank
builds and contracts K(x, x*) over its own rows; the chunks' solves and one all-reduce) for the variance and the
covariance against the single-GPU bgp_hodlr_predict on rank 0, on the prior's scale.  The grad_predict leg runs the
collective predictive_grad (the same row split for the variance gradient; two all-reduces, var's as predict's) against
the single-GPU bgp_hodlr_predict_grad on rank 0, and checks on every rank that its var is the collective predictive's
"var" bit for bit.  The symmetric-factor leg builds K~ = W W^T collectively (each rank its sub-tree's rows, one
all-gather of the top columns' rows, the top nodes on every rank) and applies W and W^T to replicated columns, against
the single-GPU factor on rank 0, and checks that every rank returns the same W Z."""
import os, sys, json
import numpy as np
import torch
import torch.distributed as dist
sys.path.insert(0, ".")
from george_b200 import kernels, _lib
from george_b200.parallel import ShardedHODLRSolver
from george_b200.solvers._hodlr import HODLRSolver
from george_b200.solvers.basic import BasicSolver

rank = int(os.environ["RANK"]); local = int(os.environ["LOCAL_RANK"]); world = int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(local)
_lib.check(_lib.load().bgp_set_device(local))
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
ok = True
for name, kernel, n, ms, exhaust in [
    ("expsq", 1.0 * kernels.ExpSquaredKernel(1.0), 20000, 100, "dense"),
    ("m32", 1.0 * kernels.Matern32Kernel(1.0), 16384, 256, "lowrank"),
    ("odd", 1.0 * kernels.ExpSquaredKernel(1.0), 8191, 100, "dense"),
    ("m32dense", 1.0 * kernels.Matern32Kernel(1.0), 6000, 100, "dense"),   # big-rank (blocked LU) top levels
    ("cfg5", 1.0 * kernels.ExpSquaredKernel(1.0) + 0.5 * kernels.ExpSine2Kernel(gamma=1.0, log_period=np.log(3.0)), 32768, 100, "lowrank"),
    ("m32big", 1.0 * kernels.Matern32Kernel(1.0), 262144, 256, "lowrank"),
]:
    rng = np.random.default_rng(1234)
    x = np.sort(rng.uniform(0, 10 * n / 1000, n)); yerr = 0.1 * np.ones(n); y = np.sin(x) + 0.1 * rng.normal(size=n)
    sh = ShardedHODLRSolver(kernel, min_size=ms, tol=1e-10, seed=42, exhaust=exhaust)
    sh.compute(x[:, None], yerr)
    ld, ds = sh.log_determinant, sh.dot_solve(y)
    a = sh.apply_inverse(y)[:, 0]
    which = np.ones(len(kernel.get_parameter_vector(include_frozen=True)), dtype=np.uint32)
    ga, gg, gd = sh.grad_terms(y, which)  # collective
    xs = np.random.default_rng(7).uniform(x.min() - 0.5, x.max() + 0.5, (300, 1))
    pv, pc = sh.predictive(kernel, xs, "var"), sh.predictive(kernel, xs, "cov")  # collective
    gv, gdv = sh.predictive_grad(kernel, xs)  # collective
    var_bits = bool(np.array_equal(gv, pv))
    ok = ok and var_bits
    Z = np.random.default_rng(9).standard_normal((n, 65))
    try:  # a level rank above the factor's limit is rejected on every rank alike (collective status)
        wz, wtz, sld = sh.apply_symmetric_factor(Z), sh.apply_symmetric_factor(Z, transpose=True), sh.symmetric_log_determinant
    except ValueError:
        wz = None
    sym_same = True
    if wz is not None:
        got = torch.from_numpy(np.ascontiguousarray(wz)).cuda()
        first = got.clone()
        dist.broadcast(first, src=0)
        sym_same = bool(torch.equal(got, first))  # every rank returns the same W Z
    ok = ok and sym_same
    if rank == 0:
        s = HODLRSolver(); s.compute(kernel, x[:, None], yerr, min_size=ms, tol=1e-10, seed=42, exhaust=exhaust)
        ld1, ds1 = s.log_determinant, s.dot_solve(y)
        a1 = s.apply_inverse(y)[:, 0]
        ga1, gg1, gd1 = np.empty(n), np.zeros(which.size), np.empty(n)
        _lib.check(s._lib.bgp_hodlr_grad_terms(s._ptr, _lib.ptr(which), _lib.ptr(y), _lib.ptr(ga1), _lib.ptr(gg1), _lib.ptr(gd1)))
        pv1 = BasicSolver._predictive_call(s._lib.bgp_hodlr_predict, s._ptr, kernel, xs, "var")
        pc1 = BasicSolver._predictive_call(s._lib.bgp_hodlr_predict, s._ptr, kernel, xs, "cov")
        kss = np.max(np.abs(kernel.get_value(xs)))
        p_rel = float(max(np.max(np.abs(pv - pv1)), np.max(np.abs(pc - pc1))) / kss)
        gv1, gdv1 = BasicSolver._predictive_grad_call(s._lib.bgp_hodlr_predict_grad, s._ptr, kernel, xs)
        pg_rel = float(max(np.max(np.abs(gv - gv1)), np.max(np.abs(gdv - gdv1))) / kss)
        g_rel = float(np.max(np.abs(gg - gg1) / np.maximum(1.0, np.abs(gg1))))
        d_rel = float(np.linalg.norm(gd - gd1) / np.linalg.norm(gd1))
        good = abs(ld - ld1) <= 1e-10 * abs(ld1) and abs(ds - ds1) <= 1e-9 * abs(ds1) and np.linalg.norm(a - a1) <= 1e-9 * np.linalg.norm(a1)
        good = good and g_rel <= 1e-9 and d_rel <= 1e-9 and np.linalg.norm(ga - ga1) <= 1e-9 * np.linalg.norm(ga1)
        good = good and p_rel <= 1e-9 and pg_rel <= 1e-9 and var_bits
        sym_rel = sym_ld_rel = None
        if wz is not None:
            wz1, wtz1, sld1 = s.apply_symmetric_factor(Z), s.apply_symmetric_factor(Z, transpose=True), s.symmetric_log_determinant
            sym_rel = float(max(np.max(np.abs(wz - wz1)) / np.max(np.abs(wz1)), np.max(np.abs(wtz - wtz1)) / np.max(np.abs(wtz1))))
            sym_ld_rel = abs(sld - sld1) / abs(sld1)
            good = good and sym_rel <= 1e-10 and sym_ld_rel <= 1e-10 and sym_same
        ok = ok and good
        print(json.dumps({"case": name, "world": world, "logdet_sharded": ld, "logdet_single": ld1, "dot_sharded": ds, "dot_single": ds1,
                          "solve_relerr": float(np.linalg.norm(a - a1) / np.linalg.norm(a1)), "grad_relerr": g_rel,
                          "grad_diag_relerr": d_rel, "predict_relerr": p_rel, "grad_predict_relerr": pg_rel,
                          "grad_predict_var_is_predict": var_bits, "sym_apply_relerr": sym_rel, "sym_logdet_relerr": sym_ld_rel,
                          "sym_apply_same_on_every_rank": sym_same, "ok": bool(good)}))
dist.barrier()
if rank == 0:
    print("MGPU_CHECK", "PASS" if ok else "FAIL")
dist.destroy_process_group()
