/*
 * bgp.h — C ABI of the H100-native GP covariance engine (libbgp_b200.so).
 *
 * This is the drop-in boundary for ONE path of dfm/george:
 *     gp.compute(x, yerr) + gp.log_likelihood(y) (+ gp.predict on the same factorisation)
 * i.e. kernel-matrix build -> factorisation (dense Cholesky | HODLR) -> log-det -> solve -> quadratic form.
 *
 * Every entry point is `extern "C"`, takes plain pointers and sizes, returns an int status
 * (0 = BGP_OK) and never lets a C++ exception cross the boundary; the message for the last
 * failing call on the calling thread is available from bgp_last_error().
 *
 * Each function names the reference interface it replaces (paths relative to the dfm/george
 * checkout, commit b5023758).  Host pointers are borrowed for the duration of a call only
 * (the reference copies its inputs as well: src/george/solvers/_hodlr.cpp:71-81,156-164).
 * Pointers are HOST pointers unless the name ends in `_dev`.
 */
#ifndef BGP_B200_H_
#define BGP_B200_H_

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------
 * Status codes.  The Python host maps them to the exception types the reference raises
 * (SURVEY.md §8b "Errors"): DIM -> RuntimeError (george::dimension_mismatch, exceptions.h:8-12),
 * NOT_COMPUTED -> RuntimeError (exceptions.h:14-18), INVALID -> ValueError (std::invalid_argument,
 * parser.h:16,33,505), INDEX -> IndexError (_hodlr.cpp:26), LINALG -> numpy.linalg.LinAlgError
 * (what scipy.linalg.cholesky raises, solvers/basic.py:68).
 * ------------------------------------------------------------------------------------------ */
enum {
  BGP_OK = 0,
  BGP_ERR_INVALID = 1,       /* malformed kernel program / argument                              */
  BGP_ERR_DIM = 2,           /* dimension mismatch between x and the kernel                      */
  BGP_ERR_NOT_COMPUTED = 3,  /* solve before compute                                             */
  BGP_ERR_LINALG = 4,        /* matrix not positive definite (or not finite): dense factorisations, *
                              * draws, and the HODLR symmetric factor (bgp_hodlr_sym_factor)      */
  BGP_ERR_CUDA = 5,          /* CUDA runtime failure; no CPU fallback exists                     */
  BGP_ERR_NO_DEVICE = 6,     /* no sm_90 device visible: the library refuses to run              */
  BGP_ERR_RANK_CAPACITY = 7, /* ACA rank exceeded the configured capacity (see bgp_hodlr_opts_t) */
  BGP_ERR_INDEX = 8,
  BGP_ERR_NOMEM = 9
};

const char* bgp_last_error(void);
/* Library/ABI version (major*1000+minor). */
int bgp_version(void);
/* Number of visible CUDA devices with compute capability 10.x; 0 if none (never an error). */
int bgp_device_count(void);
/* Select the CUDA device used by subsequently created handles of the calling thread. */
int bgp_set_device(int device);
/* Count of kernel launches issued by this library since process start (bench.py "gpu_launches"). */
uint64_t bgp_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * Kernel program: the POD form of the Python kernel-spec tree that the reference walks with
 * pybind11 attribute reads (src/george/include/george/parser.h:14-509).  Nodes are in POSTFIX
 * order (operands before their operator), so the flattened hyper-parameter vector is the
 * concatenation over leaves in program order — the order Operator::set_parameter uses
 * (kernels.h:56-69) — with, inside a stationary leaf, the kernel's own parameters first and the
 * metric parameters after them (kernels.h:1870-1875, size() at kernels.h:2005).
 * ------------------------------------------------------------------------------------------ */
#define BGP_MAX_DIM 8      /* max axes a kernel leaf may act on                                  */
#define BGP_MAX_METRIC 36  /* BGP_MAX_DIM*(BGP_MAX_DIM+1)/2 packed-Cholesky entries (metrics.h:166-168) */
#define BGP_MAX_NODES 32   /* max nodes (leaves + operators) of one program                       */
/* Limits of a kernel program on the device (BGP_ERR_INVALID past them; the Python layer raises ValueError):
 *   - at most 16 leaves (hence at most 31 nodes in use);
 *   - an expression depth of at most 8: the operand stack of the postfix program, e.g. 8 leaves nested to the right,
 *     k1 + (k2 + (... + k8)), while any number of left-nested operators keep it at 2;
 *   - hyper-parameter gradients (bgp_kmat_gradient_*, bgp_kmat_gradient_contract, bgp_dense_grad_terms,
 *     bgp_dense_batch_grad_terms, bgp_hodlr_grad_terms, bgp_*_loo_terms, bgp_dense_batch_fisher_terms) take at most 64
 *     hyper-parameters, checked before anything is solved;
 *   - input-coordinate gradients (bgp_kmat_x1/x2_gradient_general) take at most BGP_MAX_DIM = 8 input dimensions;
 *   - the HODLR solver takes at most 32 input dimensions.
 * The kernel-matrix builds, the matvec, the dense solver, the batched paths and predictions have no input-dimension
 * limit: a leaf acts on at most BGP_MAX_DIM axes, but a program's leaves may read any columns of a wider x. */

enum { BGP_OP_KERNEL = 0, BGP_OP_SUM = 1, BGP_OP_PRODUCT = 2 }; /* kernels.py:234-247 operator_type+1 */

/* kernel_type ids are the reference's (kernels.py: kernel_type attributes; parser.h:40-505). */
enum {
  BGP_K_LINEAR = 0, BGP_K_RATIONAL_QUADRATIC = 1, BGP_K_EXP = 2, BGP_K_LOCAL_GAUSSIAN = 3,
  BGP_K_EMPTY = 4, BGP_K_COSINE = 5, BGP_K_MATERN52 = 6, BGP_K_EXP_SINE2 = 7, BGP_K_CONSTANT = 8,
  BGP_K_EXP_SQUARED = 9, BGP_K_MATERN32 = 10, BGP_K_POLYNOMIAL = 11, BGP_K_DOT_PRODUCT = 12,
  /* user kernels compiled in from kernels/*.yml by tools/generate_kernels.py (the reference's generate_kernels.py:10-42
   * / docs/tutorials/new-kernel.rst): entry i of the sorted file list has id BGP_K_USER0 + i */
  BGP_K_USER0 = 13
};
enum { BGP_METRIC_NONE = -1, BGP_METRIC_ISOTROPIC = 0, BGP_METRIC_AXIS_ALIGNED = 1, BGP_METRIC_GENERAL = 2 };

typedef struct bgp_kernel_node {
  int32_t op;           /* BGP_OP_*                                                              */
  int32_t kernel_type;  /* BGP_K_* (leaf only)                                                   */
  int32_t metric_type;  /* BGP_METRIC_* ; NONE for the non-stationary kernels                    */
  int32_t ndim;         /* dimension of the input space                                          */
  int32_t naxes;        /* number of axes the leaf acts on (subspace.h:10-25)                    */
  int32_t blocked;      /* stationary kernels: block mask active (kernels.h:1897-1905)           */
  int32_t n_params;     /* number of the kernel's own hyper-parameters (excl. metric)            */
  int32_t n_metric;     /* number of metric parameters (1 | naxes | naxes(naxes+1)/2)            */
  int32_t axes[BGP_MAX_DIM];
  /* raw Python-side values, exactly what parser.h passes to the constructors:
   *   Linear: {log_gamma2, order}   RationalQuadratic: {log_alpha}   LocalGaussian: {location, log_width}
   *   Cosine: {log_period}   ExpSine2: {gamma, log_period}   Constant: {log_constant}
   *   Polynomial: {log_sigma2, order}   (order is a constant, not a hyper-parameter)                  */
  double params[4];
  double metric[BGP_MAX_METRIC];    /* metric.get_parameter_vector(include_frozen=True) (parser.h:111-116) */
  double min_block[BGP_MAX_DIM];
  double max_block[BGP_MAX_DIM];
} bgp_kernel_node_t;

typedef struct bgp_kernel_spec {
  int32_t n_nodes;
  int32_t ndim;
  bgp_kernel_node_t nodes[BGP_MAX_NODES];
} bgp_kernel_spec_t;

/* Validate a program (stack discipline, ids, dimensions).  Replaces the checks in parser.h:16-37,505. */
int bgp_spec_validate(const bgp_kernel_spec_t* spec);
/* Total number of hyper-parameters = Kernel::size() (kernels.h:56, 2005). */
int bgp_spec_num_params(const bgp_kernel_spec_t* spec, int* n_params);
/* Diagnostics: which evaluator the library picks for a program (host only, no device needed; changes nothing).
 *   out[0] the 1-D program shape of the specialised evaluators (csrc/kernel_eval.cuh BGP_SHAPE_*, 0 = interpreter),
 *          used by the ACA, the HODLR leaves, the matvec and the x1-gradient contraction;
 *   out[1] 1 when the interpreter takes its 1-D shortcut (every leaf a function of x1 - x2 on one input dimension);
 *   out[2] the profile of the kernel-matrix builds' specialised evaluator (BGP_SHAPE_EXPSQ..EXP, 0 = interpreter),
 *   out[3] its number of input dimensions, out[4] 1 for an axis-aligned metric, 0 for an isotropic one.
 * BGP_KMAT_GENERIC, which turns the specialised kernel-matrix builds off, is not reflected in out[2..4]. */
int bgp_spec_paths(const bgp_kernel_spec_t* spec, int32_t* out /* 5 */);

/* ------------------------------------------------------------------------------------------
 * Kernel-matrix build.  Replaces KernelInterface::value_symmetric / value_general / value_diagonal
 * (src/george/kernel_interface.cpp:62-77, 47-60, 79-90) and gradient_symmetric / gradient_general
 * (kernel_interface.cpp:109-125, 92-107).  x1: (n1, ndim) row-major f64; out row-major f64.
 * `which` (n_params uint32) selects the hyper-parameters to differentiate; unselected slices are 0.
 * The *_dev variants take device pointers and run on the handle-less default stream of the
 * calling thread's device; they are what the solvers call internally.
 * ------------------------------------------------------------------------------------------ */
int bgp_kmat_symmetric(const bgp_kernel_spec_t* spec, const double* x, int64_t n, double* out /* n*n */);
int bgp_kmat_general(const bgp_kernel_spec_t* spec, const double* x1, int64_t n1, const double* x2, int64_t n2,
                     double* out /* n1*n2 */);
int bgp_kmat_diagonal(const bgp_kernel_spec_t* spec, const double* x1, const double* x2, int64_t n,
                      double* out /* n */);
int bgp_kmat_gradient_symmetric(const bgp_kernel_spec_t* spec, const uint32_t* which, const double* x, int64_t n,
                                double* out /* n*n*n_params */);
int bgp_kmat_gradient_general(const bgp_kernel_spec_t* spec, const uint32_t* which, const double* x1, int64_t n1,
                              const double* x2, int64_t n2, double* out /* n1*n2*n_params */);
/* d k(x1_i, x2_j) / d x1_i  and  / d x2_j  — kernel_interface.cpp:127-141 (x1_gradient_general) and 143-157
 * (x2_gradient_general).  out[(i*n2 + j)*ndim + q]. */
int bgp_kmat_x1_gradient_general(const bgp_kernel_spec_t* spec, const double* x1, int64_t n1, const double* x2,
                                 int64_t n2, double* out /* n1*n2*ndim */);
int bgp_kmat_x2_gradient_general(const bgp_kernel_spec_t* spec, const double* x1, int64_t n1, const double* x2,
                                 int64_t n2, double* out /* n1*n2*ndim */);
/* device-resident build: out_dev[i*ld + j] (row-major, ld >= n2); diag_add_dev (may be NULL, symmetric only)
 * is added on the diagonal — the fusion of solvers/basic.py:64-65. */
int bgp_kmat_symmetric_dev(const bgp_kernel_spec_t* spec, const double* x_dev, int64_t n, const double* diag_add_dev,
                           double* out_dev, int64_t ld);
int bgp_kmat_general_dev(const bgp_kernel_spec_t* spec, const double* x1_dev, int64_t n1, const double* x2_dev,
                         int64_t n2, double* out_dev, int64_t ld);

/* ------------------------------------------------------------------------------------------
 * Matrix-free consumers of the covariance function (csrc/kmat_ops.cu): the kernel matrix is never formed.
 *
 * bgp_kmat_matvec: out (n1 x nrhs, column-major, ld n1) = K(x1, x2) v (n2 x nrhs, column-major, ld n2) [+ diag .* v].
 *   Replaces `np.dot(kernel.get_value(xs, x), alpha)` of GP.predict (src/george/gp.py:524-528, i.e.
 *   KernelInterface::value_general kernel_interface.cpp:47-60 followed by a host GEMV) without the (n1, n2) matrix;
 *   with x1 == x2 and diag = yerr^2 it applies the GP covariance itself (K (K^-1 y) == y round-trip checks at sizes
 *   where K cannot be stored).  `diag` may be NULL; it requires n1 == n2.
 * bgp_kmat_gradient_contract: out[p] = sum_ij A_ij dK_ij/dtheta_p for the symmetric gradient
 *   (kernel_interface.cpp:109-125) and a host matrix A (n, n) row-major: the `einsum("ijk,ij", dK, A)` of
 *   GP.grad_log_likelihood (gp.py:465-466) without the (n, n, P) tensor.  Unselected parameters (which[p] == 0) give 0.
 * ------------------------------------------------------------------------------------------ */
int bgp_kmat_matvec(const bgp_kernel_spec_t* spec, const double* x1, int64_t n1, const double* x2, int64_t n2,
                    const double* diag, const double* v, int64_t nrhs, double* out);
int bgp_kmat_matvec_dev(const bgp_kernel_spec_t* spec, const double* x1_dev, int64_t n1, const double* x2_dev,
                        int64_t n2, const double* diag_dev, const double* v_dev, int64_t nrhs, double* out_dev);
int bgp_kmat_gradient_contract(const bgp_kernel_spec_t* spec, const uint32_t* which, const double* x, int64_t n,
                               const double* A, double* out /* n_params */);
/* bgp_kmat_x1_gradient_matvec: input gradients contracted with a vector or with one column per point of x1,
 *   out[i*ndim + q] = (add_prior ? d k(x1_i, x1_i) / d x1_iq : 0) + scale * sum_j d k(x1_i, x2_j) / d x1_iq * V_ji
 * with V_ji = v[j] when ldv == 0 (one shared vector of n2 entries: GP.grad_predict's dmu with v = alpha, scale 1,
 * add_prior 0) and V_ji = v[i*ldv + j] when ldv >= n2 (column i of an n2 x n1 column-major matrix: dvar with
 * v = K^-1 K(x, x1), scale -2, add_prior 1).  The prior term is the derivative of the prior variance k(x, x), taken as
 * 2 d k(x, x2)/dx at x2 = x (every kernel is symmetric); it is 0 for stationary kernels.  Unlike
 * bgp_kmat_x1_gradient_general (the reference's values, L^-1 r for a general metric M = L L^T) the derivative is the
 * true one for every metric.  The (n1, n2, ndim) gradient tensor is never formed; partial sums are added in a fixed
 * order (no atomics), so identical calls return identical bits.  Errors: BGP_ERR_INVALID for ndim > BGP_MAX_DIM or a
 * negative size, BGP_ERR_DIM for 0 < ldv < n2.  n1 == 0 writes nothing; n2 == 0 gives the prior term alone. */
int bgp_kmat_x1_gradient_matvec(const bgp_kernel_spec_t* spec, const double* x1, int64_t n1, const double* x2,
                                int64_t n2, const double* v, int64_t ldv, double scale, int32_t add_prior,
                                double* out /* n1*ndim */);
int bgp_kmat_x1_gradient_matvec_dev(const bgp_kernel_spec_t* spec, const double* x1_dev, int64_t n1,
                                    const double* x2_dev, int64_t n2, const double* v_dev, int64_t ldv, double scale,
                                    int32_t add_prior, double* out_dev);

/* ------------------------------------------------------------------------------------------
 * Dense solver.  Replaces BasicSolver (src/george/solvers/basic.py:51-121): kernel matrix +
 * yerr^2 on the diagonal, Cholesky, log-det = 2 sum log diag, cho_solve, r @ U, dense inverse.
 * ------------------------------------------------------------------------------------------ */
typedef struct bgp_dense bgp_dense_t;
int bgp_dense_create(bgp_dense_t** out);
void bgp_dense_destroy(bgp_dense_t* h);
/* basic.py:51-70.  yerr is the standard deviation; yerr^2 is added on the diagonal. */
int bgp_dense_compute(bgp_dense_t* h, const bgp_kernel_spec_t* spec, const double* x, int64_t n, int32_t ndim,
                      const double* yerr);
int bgp_dense_computed(const bgp_dense_t* h);
int bgp_dense_log_determinant(const bgp_dense_t* h, double* out);
/* basic.py:72-87.  b: (n, nrhs) column-major with leading dimension ldb (a plain vector has nrhs=1); in place. */
int bgp_dense_apply_inverse(bgp_dense_t* h, double* b, int64_t nrhs, int64_t ldb);
/* basic.py:89-102 */
int bgp_dense_dot_solve(bgp_dense_t* h, const double* y, double* out);
/* basic.py:104-114: out = r @ U with r (nr, n) row-major, out (nr, n) row-major, U the upper factor. */
int bgp_dense_apply_sqrt(bgp_dense_t* h, const double* r, int64_t nr, double* out);
/* basic.py:116-121: out (n, n); symmetric so the order does not matter. */
int bgp_dense_get_inverse(bgp_dense_t* h, double* out);
/* Pickle support (the reference pickles its numpy factor, tests/test_pickle.py:21-36): copy the lower Cholesky
 * factor out (n*n, column-major, strictly-upper part zeroed) and load it back into a fresh handle. */
int bgp_dense_export_factor(bgp_dense_t* h, double* out);
int bgp_dense_import_factor(bgp_dense_t* h, const double* factor, int64_t n, double log_det);
/* Everything GP.grad_log_likelihood (gp.py:406-468) needs from the solver, computed on the device from the stored
 * factor, kernel and coordinates: alpha = K^-1 r (n), g[p] = sum_ij (alpha alpha^T - K^-1)_ij dK_ij/dtheta_p (n_params;
 * the caller multiplies by 0.5 and selects the unfrozen entries) and diag(alpha alpha^T - K^-1) (n, for the white-noise
 * term gp.py:452-456).  Replaces solver.get_inverse() (basic.py:116-121) + kernel.get_gradient (N x N x P on the host)
 * + einsum.  Any output pointer may be NULL.  Returns BGP_ERR_NOT_COMPUTED on a handle restored by
 * bgp_dense_import_factor (it holds no kernel / coordinates). */
int bgp_dense_grad_terms(bgp_dense_t* h, const uint32_t* which, const double* r, double* alpha_out, double* g_out,
                         double* diag_out);
/* bgp_dense_grad_terms plus the log-likelihood's gradient with respect to the training inputs (GP.grad_log_likelihood_x):
 *   dx_out[i * ndim + q] = sum_j (alpha alpha^T - K^-1)_ij d k(x_i, x_j) / d x_iq     (n * ndim, host)
 * the true derivative for every metric (the evaluator of bgp_kmat_x1_gradient_matvec).  Each x_i enters row i and
 * column i of K, and the 1/2 of the log-likelihood cancels the factor 2 of the symmetric pair, so dx_out is
 * d log L / d x with no further factor.  alpha_out, g_out and diag_out are bgp_dense_grad_terms' and its bits (the same
 * launches); a NULL `which` skips the parameter contraction (g_out is then not written).  K^-1 stays resident, as in
 * bgp_dense_grad_terms; after the contraction it is overwritten by alpha alpha^T - K^-1 (rounded as on the host) and
 * contracted by the x-gradient matvec with V = that matrix.  Extra device workspace: n * ndim + the matvec's partials.
 * Errors (before anything is launched): BGP_ERR_NOT_COMPUTED before compute and on a handle restored by
 * bgp_dense_import_factor; BGP_ERR_INVALID for more than BGP_MAX_DIM input dimensions and for more than 64 kernel
 * parameters with a non-NULL which. */
int bgp_dense_grad_x_terms(bgp_dense_t* h, const uint32_t* which, const double* r, double* alpha_out, double* g_out,
                           double* diag_out, double* dx_out);
/* The rows of the expected Fisher information of the hyper-parameters (GP.fisher_information), from the resident K^-1:
 * row p for each kernel parameter with which[p] != 0 (ascending p), then one row per white-noise vector v_k
 * (v: nv x n, host, row-major; dK = diag(v_k)).  With B = K^-1 dK_row K^-1 (dK_p the device program's derivative):
 *   rows_out[row * np + q] = sum_ij B_ij dK_q,ij  (np = all kernel parameters, 0 where which[q] == 0)     (nrow x np)
 *   rdiag_out[row * n + i] = B_ii                                                                        (nrow x n)
 * so F = 1/2 tr(K^-1 dK_a K^-1 dK_b) is 1/2 rows_out for kernel columns and 1/2 rdiag_out . v_l for white-noise
 * columns; the caller applies the 1/2 and symmetrises.  B runs on the FP64 tensor pipe: a kernel row materialises
 * dK_p, then T = K^-1 dK_p and B = K^-1 T^T (lower triangle, mirrored, so B is exactly symmetric); a white-noise row forms
 * K^-1 diag(v_k) K^-1 from a row-scaled copy of K^-1 in one lower product.  Each row is contracted by the parameter
 * contraction of bgp_dense_grad_terms, in a fixed order (no atomics): identical calls return identical bits.
 * With r, alpha_out / g_out / diag_out are bgp_dense_grad_terms' outputs and its bits (the same launches, first); a NULL r
 * skips alpha and the contraction of alpha alpha^T - K^-1 (those outputs are then not written).  prod_ms_out (may be
 * NULL; nrow entries) receives the device time of each row's products (the call then synchronises once per row).
 * Device workspace: K^-1 (as bgp_dense_grad_terms keeps it) + 2 n^2 (one dK_p / B buffer, one T buffer) + the products'
 * split-K slices (at most 1 GiB) + nrow * (n + np): it does not grow with the number of parameters.
 * Errors (before anything is launched): BGP_ERR_NOT_COMPUTED as bgp_dense_grad_terms; BGP_ERR_INVALID for more than
 * 64 kernel parameters, a NULL which with kernel parameters, nv < 0, a NULL v with nv > 0 and a NULL rows_out or
 * rdiag_out. */
int bgp_dense_fisher_terms(bgp_dense_t* h, const uint32_t* which, const double* r, const double* v, int32_t nv,
                           double* alpha_out, double* g_out, double* diag_out, double* rows_out, double* rdiag_out,
                           double* prod_ms_out);
/* Leave-one-out cross-validation terms (GP.loo_predict, GP.loo_log_likelihood, GP.grad_loo_log_likelihood; Rasmussen &
 * Williams, GPML eqs. 5.10-5.13), computed on the device from the stored factor, kernel and coordinates:
 *   alpha_out = K^-1 r (n),  d_out = diag(K^-1) (n)                                        (pass 1)
 *   beta_out  = K^-1 (alpha / d) (n),
 *   g_out[p]  = sum_ij A_ij dK_ij/dtheta_p (n_params; 0 where which[p] = 0; no factor 1/2: it is inside A),
 *   diag_out  = diag(A) = alpha o beta - diag(K^-1 diag(c) K^-1) (n, for the white-noise term)   (pass 2)
 * with c_i = (1 + alpha_i^2 / d_i) / (2 d_i) and A = 1/2 (beta alpha^T + alpha beta^T) - K^-1 diag(c) K^-1.  The LOO
 * predictive of y_i is mean y_i - alpha_i / d_i and variance 1 / d_i.  Any output pointer may be NULL; when beta_out,
 * g_out and diag_out are all NULL only pass 1 runs.  K^-1 is formed whole and K^-1 diag(c) K^-1 = G^T G, G =
 * diag(sqrt(c)) K^-1, runs on the FP64 tensor pipe.  Device workspace (doubles): n^2 (K^-1, kept by the handle as
 * bgp_dense_grad_terms keeps it) in pass 1; pass 2 adds n^2 for A and the product's split-K slices, n^2 each: none once
 * the product has one slice, ceil(n / 128)^2 >= 2 x the SM count (from n = 2049 on a 132-SM H100 SXM; 2 n^2 in all:
 * about 34.5 GB at n = 46411, beside the n^2 of the factor), at most four below (6 n^2), plus ceil(n / 32)^2 P for the
 * contraction and 5 n + 64.  Errors: BGP_ERR_NOT_COMPUTED before compute and on a handle restored by
 * bgp_dense_import_factor; BGP_ERR_INVALID, when pass 2 is asked for, for more than 64 kernel parameters (before
 * anything is launched) and for a d_j that is not finite and positive (the message names j; alpha_out and d_out are
 * written, pass 2 does not run). */
int bgp_dense_loo_terms(bgp_dense_t* h, const uint32_t* which, const double* r, double* alpha_out, double* d_out,
                        double* beta_out, double* g_out, double* diag_out);
/* timing of the last compute: [0]=kernel-matrix build ms, [1]=potrf ms (device events). */
int bgp_dense_last_timing(const bgp_dense_t* h, double* ms2);

/* ------------------------------------------------------------------------------------------
 * Predictive variance / covariance on the stored factorisation: gp.py:534-545 (GP.predict with return_var /
 * return_cov) without K(x*, x) or K^-1 K(x, x*) on the host.  spec = the kernel for K(x*, x) and K(x*, x*)
 * (GP.predict's `kernel`, not necessarily the factorised one), xs (ns x ndim row-major, host).
 *   VAR: out[ns]         = k(x*_j, x*_j) - Kxs_j . (K^-1 Kxs^T)_j
 *   COV: out[i*ns + j]   = K**(i,j) - sum_k Kxs(i,k) (K^-1 Kxs^T)(k,j)   (row-major, the reference's orientation)
 * K(x, x*) is built exactly as bgp_kmat_general builds K(x*, x), k(x*_j, x*_j) as bgp_kmat_diagonal and K** as
 * bgp_kmat_symmetric.  The test points are streamed in chunks of c columns on the handle's stream; c fills a 1 GiB
 * budget (c = max(64, 2^27 / N) rounded down to a multiple of 64; BGP_PREDICT_CHUNK overrides it, rounded up to a
 * multiple of 64 for HODLR).  Dense: W = L^-1 K(x, x*) (forward substitution only), var = k** - ||W_j||^2,
 * cov = K** - W^T W (lower triangle, mirrored: exactly symmetric).  HODLR: W = K_h^-1 K(x, x*) in the 64-column groups
 * of bgp_hodlr_apply_inverse (the same W as apply_inverse), var = k** - B_j . W_j, cov = K** - B^T W.  The reductions
 * add in a fixed order (no atomics), so identical calls return identical bits as far as the solve does: the HODLR solve
 * accumulates a node's Gram product with atomics once a half has more than 512 rows.  Negative variances are returned
 * as computed.
 * Device workspace (doubles), besides the result (ns or ns^2) and xs:
 *   dense VAR  N*c + O(c)                 dense COV  N*ns + split-K slices (ns^2 each, at most 2^27 in all)
 *   HODLR VAR  2*N*c + O(c)               HODLR COV  N*ns + N*c + split-K slices (c*ns each, at most 2^27 in all)
 * A product of one split-K slice (at least two 128 x 128 tiles per SM, N <= 256, or more than 2^26 entries) has no
 * slice buffer: it is subtracted from the result in place.
 * Errors: BGP_ERR_NOT_COMPUTED before compute and on a dense handle restored by bgp_dense_import_factor (no
 * coordinates); BGP_ERR_DIM when the spec's ndim differs from the handle's; BGP_ERR_INVALID on a host-exchange HODLR
 * shard, an unknown `what` or ns < 0; BGP_ERR_NOMEM when the workspace cannot be allocated.  ns == 0 writes nothing.
 * ------------------------------------------------------------------------------------------ */
enum { BGP_PREDICT_VAR = 0, BGP_PREDICT_COV = 1 };
int bgp_dense_predict(bgp_dense_t* h, const bgp_kernel_spec_t* spec, const double* xs, int64_t ns, int32_t what,
                      double* out);
/* Gradients of the predictive variance with respect to the test points (GP.grad_predict):
 *   var[j]            = bgp_*_predict's VAR output, bit for bit (the same chunks and steps);
 *   dvar[j*ndim + q]  = d var_j / d x*_jq = (d1 + d2) k(x*_j, x*_j)_q - 2 sum_i d k(x*_j, x_i) / d x*_jq W_ij
 * with W = K^-1 K(x, x*) per chunk: dense, the backward sweep L^-T applied in place to the chunk's L^-1 K(x, x*) once
 * var is reduced; HODLR, the chunk's K_h^-1 K(x, x*) of the VAR path.  The contraction is bgp_kmat_x1_gradient_matvec's
 * (true derivatives for every metric), so identical calls return identical bits as far as the solve does.  Device
 * workspace: the VAR path's plus O(c * ndim).  Errors: those of bgp_*_predict, and BGP_ERR_INVALID for ndim >
 * BGP_MAX_DIM and on a host-exchange HODLR shard, all checked before anything is launched.  ns == 0 writes nothing. */
int bgp_dense_predict_grad(bgp_dense_t* h, const bgp_kernel_spec_t* spec, const double* xs, int64_t ns, double* var,
                           double* dvar);

/* ------------------------------------------------------------------------------------------
 * Batched log-likelihood terms (GP.batch_log_likelihood): B parameter vectors of one kernel program on the same x,
 * e.g. the walkers of one ensemble-sampler step.
 * For b in [0, B): K_b = K(x, x; spec with its parameter slots replaced by params[b*P .. b*P+P)) + diag(yerr[b]^2),
 * lower Cholesky, log_det[b] = log|K_b|, quad[b] = r_b^T K_b^-1 r_b.  info[b] = 0, or the leading-minor index k+1
 * exactly as bgp_dense_compute reports it (log_det / quad then NaN), or -1 when member b's program fails the
 * validation bgp_dense_compute applies.  x (n x ndim row-major), yerr and r (B x n row-major), all host memory.
 * The parameter slots are, leaf by leaf in node order, the leaf's params[0 .. own parameter count) followed by its
 * metric[0 .. n_metric): the order of bgp_spec_num_params, and of Kernel.get_parameter_vector(include_frozen=True).
 * Each member's matrix, factor and log_det are bit-identical to bgp_dense_compute with the member's spec and yerr;
 * quad is summed in a fixed order (bgp_dense_dot_solve adds per-CTA partials atomically), so a member's results do
 * not depend on B, its position or the chunking.  Members run in chunks of as many n x n matrices as fit in 4 GiB of
 * device memory (BGP_BATCH_CHUNK=<members> overrides it); every step of a chunk is one launch for all its members.
 * Device workspace: chunk * (n^2 + 5 n) doubles + B programs, kept by the handle for the next call.
 * Errors: BGP_ERR_INVALID for n <= 0, B < 0, a malformed template or P != bgp_spec_num_params(spec); BGP_ERR_DIM
 * when the kernel's ndim differs from ndim; BGP_ERR_NOMEM when a single member does not fit.  A member that is not
 * positive definite is not an error.  B == 0 writes nothing.
 * ------------------------------------------------------------------------------------------ */
typedef struct bgp_dense_batch bgp_dense_batch_t;
int bgp_dense_batch_create(bgp_dense_batch_t** out);
void bgp_dense_batch_destroy(bgp_dense_batch_t* h);
int bgp_dense_batch_log_likelihood(bgp_dense_batch_t* h, const bgp_kernel_spec_t* spec, const double* params,
                                   int64_t B, int64_t P, const double* x, int64_t n, int32_t ndim,
                                   const double* yerr, const double* r,
                                   double* log_det, double* quad, int32_t* info);
/* Batched gradient terms (GP.batch_grad_log_likelihood): for the same B members as bgp_dense_batch_log_likelihood
 * (spec, params, x, yerr; r = y - mean(x) per member, B x n row-major) and one selection `which` (P entries, shared by
 * all members), what bgp_dense_grad_terms returns for each member plus its log-likelihood terms:
 *   log_det[b], quad[b]    as bgp_dense_batch_log_likelihood computes them (bit-identical to it)
 *   alpha[b*n + i]         (K_b^-1 r_b)_i
 *   g[b*P + p]             sum_ij (alpha_b alpha_b^T - K_b^-1)_ij dK_b,ij/dtheta_p   (zeros where which[p] == 0)
 *   diag[b*n + i]          (alpha_b alpha_b^T - K_b^-1)_ii
 * Any output but info may be NULL.  Each member's alpha, g, diag and log_det are bit-identical to bgp_dense_compute
 * followed by bgp_dense_grad_terms on member b's spec and yerr: the same kernels run with a member index (K_b^-1 by
 * solving against the identity, through the few-column solve when n <= 8, and the same contraction tiles and fixed
 * reduction order), so a member's results do not depend on B, its position or the chunking.  info[b] as in
 * bgp_dense_batch_log_likelihood (0, the leading-minor index, or -1 for an invalid member program); a failed member's
 * outputs are NaN and do not disturb the other members.
 * Members run in chunks that fit in 4 GiB of device memory (BGP_BATCH_CHUNK=<members> overrides it); every step of a
 * chunk is one launch for all its members.  Device workspace per member (doubles): 2 n^2 (factor and K^-1) +
 * (4 + t) n (t = n for n <= 8, else 1) + ceil(n / 32)^2 P contraction partials + P.  Shared: B programs, x, which.
 * Forming K_b^-1 costs about 2 n^3 flops per member on the CUDA cores, against n^3 / 3 for the factorisation.
 * Errors: those of bgp_dense_batch_log_likelihood; BGP_ERR_INVALID for P > 64, before anything is solved.  B == 0
 * writes nothing. */
int bgp_dense_batch_grad_terms(bgp_dense_batch_t* h, const bgp_kernel_spec_t* spec, const double* params,
                               int64_t B, int64_t P, const double* x, int64_t n, int32_t ndim,
                               const double* yerr, const double* r,      /* B x n row-major          */
                               const uint32_t* which,                    /* P, shared by all members */
                               double* log_det, double* quad,            /* B, may be NULL           */
                               double* alpha, double* diag,              /* B x n, may be NULL       */
                               double* g,                                /* B x P, may be NULL       */
                               int32_t* info);                           /* B                        */
/* Batched leave-one-out terms (GP.batch_loo_predict, GP.batch_loo_log_likelihood, GP.batch_grad_loo_log_likelihood):
 * for the same B members as bgp_dense_batch_log_likelihood (spec, params, x, yerr; r = y - mean(x) per member, B x n
 * row-major), what bgp_dense_loo_terms returns for each member:
 *   alpha[b*n + i]   (K_b^-1 r_b)_i                    d[b*n + i]      (K_b^-1)_ii                         (pass 1)
 *   beta[b*n + i]    (K_b^-1 (alpha_b / d_b))_i        g[b*P + p]      sum_ij A_b,ij dK_b,ij/dtheta_p      (pass 2)
 *   diag[b*n + i]    A_b,ii
 * with A_b and c_b as in bgp_dense_loo_terms.  which == NULL runs pass 1 only, with no parameter limit; beta, g and
 * diag may then be NULL.  which != NULL (P entries, shared by all members) runs pass 2 for every member; any output
 * but info may be NULL.  Each member's outputs are bit-identical to bgp_dense_compute followed by bgp_dense_loo_terms
 * on member b's spec and yerr: the same kernels run with a member index (K_b^-1 by solving against the identity,
 * through the few-column solve when n <= 8; the G^T G product with the single call's split-K plan; the same contraction
 * tiles and fixed reduction order), so a member's results do not depend on B, its position or the chunking.
 * info[b] as in bgp_dense_batch_log_likelihood (0, the leading-minor index, or -1 for an invalid member program); a
 * failed member's outputs are NaN and do not disturb the other members.  Unlike bgp_dense_loo_terms nothing checks d on
 * the host between the passes: a member whose d is not finite and positive is not an error, its pass-2 rows are what
 * that arithmetic gives, and the caller checks d (GP does, raising the single call's ValueError).
 * Members run in chunks that fit in 4 GiB of device memory (BGP_BATCH_CHUNK=<members> overrides it), capped so that
 * the split-K product is one launch; every step of a chunk is one launch for all its members, with no host work in
 * between, so the launch count depends on n and the number of chunks, never on B within a chunk.
 * Device workspace per member (doubles): 2 n^2 (factor and K^-1) + (4 + t) n (t = n for n <= 8, else 1); pass 2 adds
 * n^2 (A) + nsplit n^2 (the product's split-K slices, none when nsplit = 1: 2 n^2 at n = 512, none from n = 2049 on a
 * 132-SM H100 SXM) + 2 n (beta, c) + ceil(n / 32)^2 P contraction partials + P.  Shared: B programs, x, which.
 * Errors: those of bgp_dense_batch_log_likelihood; BGP_ERR_INVALID for P > 64 when which != NULL, before anything is
 * launched; BGP_ERR_NOMEM when a single member does not fit.  B == 0 writes nothing. */
int bgp_dense_batch_loo_terms(bgp_dense_batch_t* h, const bgp_kernel_spec_t* spec, const double* params,
                              int64_t B, int64_t P, const double* x, int64_t n, int32_t ndim,
                              const double* yerr, const double* r,     /* B x n row-major             */
                              const uint32_t* which,                   /* P, or NULL for pass 1 only  */
                              double* alpha, double* d,                /* B x n, may be NULL          */
                              double* beta, double* g, double* diag,   /* B x n, B x P, B x n, or NULL */
                              int32_t* info);                          /* B                           */
/* Batched Fisher information rows (GP.batch_fisher_information): for the same B members as
 * bgp_dense_batch_log_likelihood (spec, params, x, yerr) and one selection `which` (P entries, shared by all members),
 * what bgp_dense_fisher_terms returns for each member, plus the mean block's solve:
 *   alpha[b*n + i], g[b*P + p], diag[b*n + i]   bgp_dense_batch_grad_terms' outputs, with r (B x n row-major)
 *   rows[(b*nrow + k)*P + q]                      sum_ij B_b,k,ij dK_b,ij/dtheta_q                        (B x nrow x P)
 *   rdiag[(b*nrow + k)*n + i]                     B_b,k,ii                                                (B x nrow x n)
 *   kdmu[(b*nm + m)*n + i]                        (K_b^-1 dmu_b,m)_i                                      (B x nm x n)
 * with nrow = (number of which[q] != 0) + nv and B_b,k = K_b^-1 dK K_b^-1 for row k's dK, in bgp_dense_fisher_terms'
 * order: the kernel rows (ascending q), then one row per white-noise vector v[(b*nv + k)*n + i] (B x nv x n: the vectors
 * depend on the member's white-noise parameters; dK = diag(v_b,k)).  dmu (B x nm x n) holds each member's nm mean
 * gradients; kdmu is the nm-column bgp_dense_apply_inverse of them.  A NULL r skips the residual upload, alpha and the
 * contraction of alpha alpha^T - K^-1 (alpha, g and diag are then not written).  Any output but info may be NULL.
 * Each member's outputs are bit-identical to bgp_dense_compute followed by bgp_dense_fisher_terms and
 * bgp_dense_apply_inverse(dmu_b) on member b's spec and yerr: the same kernels run with a member index (K_b^-1 by
 * solving against the identity; the gradient planes with the same evaluator and one-hot mask; both products with the
 * single call's split-K plan; the same contraction tiles and fixed reduction order), so a member's results do not depend
 * on B, its position or the chunking.  info[b] as in bgp_dense_batch_log_likelihood (0, the leading-minor index, or -1
 * for an invalid member program); a failed member's outputs are NaN and do not disturb the other members.
 * Members run in chunks that fit in 4 GiB of device memory (BGP_BATCH_CHUNK=<members> overrides it), capped so that
 * each split-K product is one launch; every launch of a row covers the whole chunk, so the launch count depends on n,
 * nrow and the number of chunks, never on B within a chunk.
 * Device workspace per member (doubles): 2 n^2 (factor and K^-1) + 2 n^2 (P and T, none when nrow = 0) + nsplit n^2
 * (the products' split-K slices, none when nsplit = 1: 2 n^2 at n = 512, none from n = 2049 on a 132-SM H100 SXM) +
 * (4 + t) n (the vectors of batch_reserve_common; t = the larger of n for n <= 8 and nm for nm <= 8, else 1) +
 * ceil(n / 32)^2 P contraction partials + P (g) + nrow (P + n) (rows, rdiag) + nv n (v) + nm n (dmu).  Shared: B
 * programs, x, which.
 * Errors: those of bgp_dense_batch_log_likelihood; BGP_ERR_INVALID for P > 64, a NULL which with P > 0, nv < 0 or nm < 0,
 * and a NULL v or dmu with nv > 0 or nm > 0, before anything is solved; BGP_ERR_NOMEM when a single member does not
 * fit.  B == 0 writes nothing. */
int bgp_dense_batch_fisher_terms(bgp_dense_batch_t* h, const bgp_kernel_spec_t* spec, const double* params,
                                 int64_t B, int64_t P, const double* x, int64_t n, int32_t ndim,
                                 const double* yerr, const double* r,   /* B x n row-major; r may be NULL */
                                 const uint32_t* which,                 /* P, shared by all members       */
                                 const double* v, int32_t nv,           /* B x nv x n                     */
                                 const double* dmu, int32_t nm,         /* B x nm x n                     */
                                 double* alpha, double* g, double* diag, /* B x n, B x P, B x n, or NULL  */
                                 double* rows, double* rdiag,           /* B x nrow x P, B x nrow x n     */
                                 double* kdmu,                          /* B x nm x n, may be NULL        */
                                 int32_t* info);                        /* B                              */
/* Batched predictions (GP.batch_predict): for the same B members as bgp_dense_batch_log_likelihood (spec, params, x,
 * yerr; r = y - mean(x) per member, B x n row-major) and the test points xs (ns x ndim row-major, host):
 *   mean[b*ns + j]        = (K_b(x*, x) K_b^-1 r_b)_j            (the kernel part of GP.predict's mean)
 *   out == NULL           mean only
 *   what == BGP_PREDICT_VAR   out[b*ns + j]        = k_b(x*_j, x*_j) - K_b(x*_j, x) K_b^-1 K_b(x, x*_j)
 *   what == BGP_PREDICT_COV   out[(b*ns + i)*ns + j] = K_b**(i, j) - K_b(x*_i, x) K_b^-1 K_b(x, x*_j)
 * Every entry is bit-identical to the single path on member b's spec and yerr: alpha = bgp_dense_apply_inverse of r_b
 * (one right-hand side), the mean = bgp_kmat_matvec(xs, x, alpha), VAR / COV = bgp_dense_predict after
 * bgp_dense_compute.  Each step runs the single path's kernels with a member index, with its split and chunk decisions
 * (test-point chunks of predict_chunk_cols(n) columns, BGP_PREDICT_CHUNK applies alike); a member's results therefore
 * do not depend on B, its position or the chunking.  info[b] as in bgp_dense_batch_log_likelihood; a failed member's
 * rows of mean and out are NaN and do not disturb the other members.
 * Members run in chunks that fit in 4 GiB of device memory (BGP_BATCH_CHUNK=<members> overrides it; a covariance chunk
 * also keeps its split-K product to one launch); every step of a chunk is one launch for all its members, so the launch
 * count depends on n, ns and the number of chunks, never on B within a chunk.
 * Device workspace per member (doubles): n^2 + (4 + t) n + ns + P_mv, t = 8 with out (the few-column solve), 1 without,
 * P_mv = nsplit_mv * ns * 4 matvec partials (nsplit_mv <= ceil(n / 512)); VAR adds n c + 2 c + P_var (c the test-point
 * chunk, P_var <= c * ceil(n / 1024) partials); COV adds n ns + ns^2 (1 + nsplit) (K** and the split-K slices,
 * nsplit * ns^2 <= max(ns^2, 2^27)).  Shared: B programs, x, xs.  The handle keeps it for the next call.
 * Errors: those of bgp_dense_batch_log_likelihood; BGP_ERR_INVALID for ns < 0 or an unknown `what` with out != NULL.
 * B == 0 writes nothing. */
int bgp_dense_batch_predict(bgp_dense_batch_t* h, const bgp_kernel_spec_t* spec, const double* params,
                            int64_t B, int64_t P, const double* x, int64_t n, int32_t ndim,
                            const double* yerr, const double* r,            /* B x n, row-major            */
                            const double* xs, int64_t ns, int32_t what,      /* BGP_PREDICT_VAR / _COV       */
                            double* mean,                                    /* B x ns                       */
                            double* out,                                     /* B x ns, B x ns x ns, or NULL */
                            int32_t* info);
/* Batched predictive gradients (GP.batch_grad_predict): for the same B members as bgp_dense_batch_predict (spec,
 * params, x, yerr, r, xs), what bgp_dense_predict_grad and the input-gradient contraction give each member:
 *   mean[b*ns + j]            as bgp_dense_batch_predict
 *   dmu[(b*ns + j)*ndim + q]  = sum_i d k_b(x*_j, x_i) / d x*_jq alpha_bi      (alpha_b = K_b^-1 r_b)
 *   with_var != 0:
 *   var[b*ns + j]             as bgp_dense_batch_predict with BGP_PREDICT_VAR
 *   dvar[(b*ns + j)*ndim + q] = 2 d1 k_b(x*_j, x*_j)_q - 2 sum_i d k_b(x*_j, x_i) / d x*_jq (K_b^-1 K_b(x, x*_j))_i
 * Every entry is bit-identical to the single path on member b's spec and yerr: bgp_dense_apply_inverse of r_b (one
 * right-hand side), bgp_kmat_matvec and bgp_kmat_x1_gradient_matvec(xs, x, alpha) for mean and dmu, bgp_dense_predict_grad
 * after bgp_dense_compute for var and dvar.  The steps of a member chunk are bgp_dense_batch_predict's (factor, alpha,
 * mean, the VAR chunks) followed by bgp_dense_predict_grad's backward sweep L_b^-T and contraction per test-point
 * chunk, each with a member index and with the single path's split and chunk decisions (test-point chunks of
 * predict_chunk_cols(n) columns, BGP_PREDICT_CHUNK applies alike; the contraction's evaluator is the one the single
 * path picks from the program's shape).  A member's results therefore do not depend on B, its position or the
 * chunking.  info[b] as in bgp_dense_batch_log_likelihood; a failed member's rows of every output are NaN and do not
 * disturb the other members.
 * Members run in chunks that fit in 4 GiB of device memory (BGP_BATCH_CHUNK=<members> overrides it); every step of a
 * chunk is one launch for all its members, so the launch count depends on n, ns, with_var and the number of chunks,
 * never on B within a chunk.
 * Device workspace per member (doubles): bgp_dense_batch_predict's (mean only without with_var, VAR with it) plus
 * ns ndim (dmu) + P_xg, and with with_var c ndim (a chunk of dvar); P_xg = nsplit * m * ndim contraction partials for
 * the larger of the m = ns (dmu) and m = c (dvar) contractions, nsplit <= ceil(n / 512).  Shared: B programs, x, xs.
 * The handle keeps it for the next call.
 * Errors: those of bgp_dense_batch_log_likelihood; BGP_ERR_INVALID for ndim > BGP_MAX_DIM (before anything else),
 * ns < 0, or with_var without var or dvar.  B == 0 writes nothing; ns == 0 factorises (info) and writes no rows. */
int bgp_dense_batch_predict_grad(bgp_dense_batch_t* h, const bgp_kernel_spec_t* spec, const double* params,
                                 int64_t B, int64_t P, const double* x, int64_t n, int32_t ndim,
                                 const double* yerr, const double* r,       /* B x n, row-major            */
                                 const double* xs, int64_t ns, int32_t with_var,
                                 double* mean,                               /* B x ns                      */
                                 double* dmu,                                /* B x ns x ndim               */
                                 double* var,                                /* B x ns, or NULL             */
                                 double* dvar,                               /* B x ns x ndim, or NULL      */
                                 int32_t* info);                             /* B                           */
/* Batched draws (GP.batch_sample_conditional): for the same B members as bgp_dense_batch_predict (spec, params, x,
 * yerr, r, xs), what bgp_dense_sample draws for each member from its predictive covariance:
 *   draws[(b*size + a)*ns + j] = mu_b[j] + sum_{i <= j} z[(b*size + a)*ns + i] L_b(j, i)
 * with mu_b = (K_b(x*, x) K_b^-1 r_b) + mean_add[b*ns + j] (the kernel part of GP.predict's mean plus the mean model at
 * x*, one IEEE add as the host sums them) and L_b the lower Cholesky factor of sym(C_b) + jitter * I, C_b the member's
 * BGP_PREDICT_COV output.  mean_add (B x ns), z (B x size x ns, the caller's standard normals) and draws are host
 * arrays.  Each member's draws are bit-identical to bgp_dense_sample(mean = bgp_kmat_matvec(xs, x, alpha) + mean_add[b])
 * on a handle computed with member b's spec and yerr: the covariance steps are bgp_dense_batch_predict's, and the
 * symmetrisation, the factorisation and the product (rows below BGP_SAMPLE_DMMA_ROWS draws, the DMMA GEMM from it with
 * one descriptor per member, 128 columns and draw slab) are bgp_dense_sample's with a member index.  A member's draws
 * therefore do not depend on B, its position or the chunking.
 *   info[b]       as bgp_dense_batch_predict reports it (0, the leading-minor index of K_b, -1 for an invalid program)
 *   draw_info[b]  0, or the leading-minor index of sym(C_b) + jitter * I (bgp_dense_sample's BGP_ERR_LINALG); 0 where
 *                 info[b] != 0
 * A failed member's draws are NaN and do not disturb the other members: its later steps run on its own slabs, and
 * nothing synchronises inside a chunk.  Members run in chunks that fit in 4 GiB of device memory (BGP_BATCH_CHUNK
 * overrides it), capped so that the split-K covariance product and the draws' DMMA product are one launch each; every
 * step of a chunk is one launch for all its members, so the launch count depends on n, ns, size and the number of
 * chunks, never on B within a chunk.
 * Device workspace per member (doubles): bgp_dense_batch_predict's with COV, plus 2 size ns + ns (z, the draws, the
 * mean).  Shared: B programs, x, xs.  The handle keeps it for the next call.
 * Errors: those of bgp_dense_batch_predict and of bgp_dense_sample's argument checks (BGP_ERR_INVALID for ns < 0,
 * size < 0, a negative or non-finite jitter).  A member that is not positive definite, in K or in the covariance, is
 * not an error.  B == 0 writes nothing; ns == 0 or size == 0 factorises (info) and draws nothing (draw_info 0). */
int bgp_dense_batch_sample(bgp_dense_batch_t* h, const bgp_kernel_spec_t* spec, const double* params,
                           int64_t B, int64_t P, const double* x, int64_t n, int32_t ndim,
                           const double* yerr, const double* r,          /* B x n                      */
                           const double* xs, int64_t ns,
                           const double* mean_add,                       /* B x ns: mean model at xs    */
                           const double* z, int64_t size, double jitter, /* B x size x ns              */
                           double* draws,                                /* B x size x ns              */
                           int32_t* info, int32_t* draw_info);

/* ------------------------------------------------------------------------------------------
 * HODLR solver.  Replaces _hodlr.HODLRSolver (src/george/solvers/_hodlr.cpp:115-204) and the
 * hodlr::Node tree behind it (src/george/include/george/hodlr.h:13-256).
 * ------------------------------------------------------------------------------------------ */
typedef struct bgp_hodlr bgp_hodlr_t;

enum {
  BGP_RNG_PER_NODE = 0, /* each tree node draws from its own mt19937 stream (level-parallel build)     */
  BGP_RNG_REFERENCE = 1 /* one mt19937 threaded through the pre-order recursion, as hodlr.h:35,58-61   */
};

typedef struct bgp_hodlr_opts {
  int32_t min_size;      /* default 100 (_hodlr.cpp:202)                                         */
  int32_t seed;          /* default 42                                                            */
  double  tol;           /* default 0.1                                                           */
  int32_t rng_mode;      /* BGP_RNG_*                                                             */
  int32_t rank_capacity; /* max columns kept per low-rank factor; 0 = automatic                   */
  /* multi-GPU sharding by top-level sub-tree (SURVEY.md §8e): this process owns sub-tree
   * `shard_rank` of `shard_count` (a power of two; 1 = whole tree).                             */
  int32_t shard_rank;
  int32_t shard_count;
  /* What to do when the ACA runs out of candidate rows (every remaining row's residual is < 1e-14):
   *   BGP_EXHAUST_DENSE   (0, default) return the dense factorisation, rank = min(rows, cols), as hodlr.h:161-176 does;
   *   BGP_EXHAUST_LOWRANK (1) keep the low-rank factors found so far: at that point EVERY row has been tested, so the
   *                        approximation is verified to 1e-14 per entry and differs from the dense answer by rounding.
   * Kernels that are exactly low rank on sorted 1-D inputs (Matern-3/2, Cosine, ...) hit this on most small nodes. */
  int32_t exhaust_mode;
} bgp_hodlr_opts_t;
enum { BGP_EXHAUST_DENSE = 0, BGP_EXHAUST_LOWRANK = 1 };

/* The reference's defaults (solvers/hodlr.py:43, _hodlr.cpp:202): min_size 100, tol 0.1, seed 42 — and, because at that
 * tolerance the result depends on the pivot order, rng_mode = BGP_RNG_REFERENCE and exhaust_mode = BGP_EXHAUST_DENSE: a
 * caller that changes nothing gets the reference's algorithm.  The level-parallel BGP_RNG_PER_NODE is the mode to choose
 * for tight tolerances (the Python plug-in does so automatically for tol <= 1e-6) and the only one that shards. */
void bgp_hodlr_default_opts(bgp_hodlr_opts_t* o);
int bgp_hodlr_create(bgp_hodlr_t** out);
void bgp_hodlr_destroy(bgp_hodlr_t* h);
/* _hodlr.cpp:55-94 (Solver::compute): snapshot kernel + x, diag = yerr^2, build and factor the tree. */
int bgp_hodlr_compute(bgp_hodlr_t* h, const bgp_kernel_spec_t* spec, const double* x, int64_t n, int32_t ndim,
                      const double* yerr, const bgp_hodlr_opts_t* opts);
/* same with x / yerr already resident on the device (bench "value" leg; inputs in HBM). */
int bgp_hodlr_compute_dev(bgp_hodlr_t* h, const bgp_kernel_spec_t* spec, const double* x_dev, int64_t n,
                          int32_t ndim, const double* yerr_dev, const bgp_hodlr_opts_t* opts);
int bgp_hodlr_computed(const bgp_hodlr_t* h);               /* _hodlr.cpp:123 */
int bgp_hodlr_log_determinant(const bgp_hodlr_t* h, double* out); /* _hodlr.cpp:124 */
/* _hodlr.cpp:156-164: b (n, nrhs) column-major, leading dimension ldb, solved in place. */
int bgp_hodlr_apply_inverse(bgp_hodlr_t* h, double* b, int64_t nrhs, int64_t ldb);
/* _hodlr.cpp:178-182 */
int bgp_hodlr_dot_solve(bgp_hodlr_t* h, const double* y, double* out);
int bgp_hodlr_dot_solve_dev(bgp_hodlr_t* h, const double* y_dev, double* out);
/* _hodlr.cpp:193-199: dense inverse (n, n). */
int bgp_hodlr_get_inverse(bgp_hodlr_t* h, double* out);

/* The HODLR counterpart of bgp_dense_grad_terms (K^-1 by solving against the identity on the device, as
 * _hodlr.cpp:193-199 does on the host).  Two regimes, with the same outputs:
 *   n <= 65536 (n^2 <= 2^32 doubles): K^-1 is formed whole (n^2 doubles of device workspace) and contracted with the
 *     kernel gradient, each unordered pair evaluated once.
 *   larger n: K^-1 is streamed in column slabs of c = max(64, 2^27 / n) columns, rounded down to a multiple of 64
 *     (1 GiB): per slab the identity columns E_J are solved with a row-restricted solve (only the leaves and nodes that
 *     meet the rows J run, bit for bit the full solve) and contracted over every ordered pair (i, j in J), so K^-1 is
 *     never resident.  Device workspace (doubles): n c + ceil(n / 32) P + ceil(n / 1024) (c / 32) P, plus 2 n + 64.
 *     The sum order depends only on n: g does not depend on c, and two identical calls return the same bits.
 * BGP_GRAD_CHUNK=<c> (environment, read at every call; rounded up to a multiple of 64) forces the streamed path at any n
 * with c-column slabs, a diagnostic switch like BGP_PREDICT_CHUNK.
 * On a sharded factorisation with a matching communicator (see the multi-GPU block below) the call is COLLECTIVE, with r
 * replicated, and always streamed: alpha by the collective solve, each shard's slabs of its own columns
 * (bgp_hodlr_grad_terms_local_dev), one all-reduce of the P doubles of g and one all-gather of the diag slices; every
 * rank returns the whole alpha, g and diag.  diag_out must be NULL on every rank or on none (it decides whether the
 * diag all-gather is issued); alpha_out and g_out only affect this rank's copies.  Errors: BGP_ERR_NOT_COMPUTED before
 * compute, BGP_ERR_INVALID for more than 64 kernel parameters (before anything is solved or exchanged) and on a
 * host-exchange shard, which computes its part with bgp_hodlr_grad_terms_local_dev instead. */
int bgp_hodlr_grad_terms(bgp_hodlr_t* h, const uint32_t* which, const double* r, double* alpha_out, double* g_out,
                         double* diag_out);
/* One shard's part of the streamed gradient: with J = this handle's own rows [row0, row0 + rows) ([0, n) unsharded),
 *   g_part_out[p] = sum_{i in [0, n), j in J} (alpha_i alpha_j - K^-1_ij) dK_ij/dtheta_p   (host, P doubles; 0 where
 *                   which[p] = 0),
 *   diag_dev[j]   = alpha_j^2 - K^-1_jj for j in J only (device, n rows; no other row is written; may be NULL),
 * from alpha_dev, the full replicated n-vector K^-1 r on the device (on a host-exchange shard: solve_local_dev, the host's
 * all-gather, solve_top_dev).  K^-1 E_J is streamed in slabs of the bgp_hodlr_grad_terms width that start at the
 * multiple of 64 at or below row0, with the identity placed in J only; each slab is solved with the row-restricted solve
 * (this shard's leaves and owned levels, then the top levels on the top panels) and contracted over J.  Issues no
 * collective, so shards may call it independently; summing the P shards' g_part_out and assembling their diag slices
 * gives the gradient.  On an unsharded handle it returns bit for bit what bgp_hodlr_grad_terms returns on the streamed
 * path with the same slab width.  g does not depend on the slab width, and two identical calls return the same bits.
 * bgp_hodlr_last_grad_timing reports this call's slabs, slab width and (profiling on) its solve and contraction times.
 * Errors: BGP_ERR_NOT_COMPUTED before compute and on a shard whose top levels are not finished; BGP_ERR_INVALID for more
 * than 64 kernel parameters and for a NULL alpha_dev (both before anything is launched). */
int bgp_hodlr_grad_terms_local_dev(bgp_hodlr_t* h, const uint32_t* which, const double* alpha_dev, double* g_part_out,
                                   double* diag_dev);
/* bgp_dense_grad_x_terms on the HODLR matrix: alpha_out, g_out, diag_out are bgp_hodlr_grad_terms' and its bits, and
 *   dx_out[i * ndim + q] = sum_j (alpha alpha^T - K~^-1)_ij d k(x_i, x_j) / d x_iq
 * with K~^-1 the inverse of the HODLR matrix and the exact kernel derivative (the hybrid that bgp_hodlr_grad_terms
 * returns for the hyper-parameters).  Resident regime (n <= 65536, BGP_GRAD_CHUNK unset): as bgp_dense_grad_x_terms.
 * Streamed regime: each slab W = K~^-1 E_J contracts, in the same kernel pass as g, the input gradient of its own
 * columns, dx_j = sum_i (alpha_i alpha_j - W_ij) d k(x_j, x_i) / d x_j (the kernel differentiated in x_j, so
 * non-stationary kernels are exact); the per-row-split partials are summed in an order that depends only on n, so dx
 * does not depend on the slab width and two identical calls return the same bits.  Extra device workspace: n * ndim +
 * ceil(n / 1024) * c * ndim.  The resident and streamed dx agree to rounding (their sums run in different orders).
 * On a sharded factorisation with a matching communicator the call is COLLECTIVE, as bgp_hodlr_grad_terms is: the
 * collective alpha solve, each shard's slabs over its own columns, the all-reduce of g, the all-gather of the diag
 * slices when diag_out is set, and one all-gather of the dx row slices; no collective sits inside the slab loop.
 * Errors (before anything is launched): BGP_ERR_NOT_COMPUTED before compute; BGP_ERR_INVALID for more than BGP_MAX_DIM
 * input dimensions, for more than 64 kernel parameters with a non-NULL which, and on a host-exchange shard (which
 * computes its part with bgp_hodlr_grad_x_terms_local_dev). */
int bgp_hodlr_grad_x_terms(bgp_hodlr_t* h, const uint32_t* which, const double* r, double* alpha_out, double* g_out,
                           double* diag_out, double* dx_out);
/* One shard's part of bgp_hodlr_grad_x_terms: bgp_hodlr_grad_terms_local_dev's g_part_out and diag_dev (its bits) and
 * dx_dev[j * ndim + q] (device, n * ndim) for the rows j of this handle only (no other row is written).  Issues no
 * collective.  On an unsharded handle it returns bit for bit what bgp_hodlr_grad_x_terms returns on the streamed path.
 * A NULL which skips the parameter contraction.  Errors (before anything is launched): BGP_ERR_NOT_COMPUTED as
 * bgp_hodlr_grad_terms_local_dev; BGP_ERR_INVALID for more than BGP_MAX_DIM input dimensions, more than 64 kernel
 * parameters with a non-NULL which, a NULL alpha_dev and a NULL dx_dev. */
int bgp_hodlr_grad_x_terms_local_dev(bgp_hodlr_t* h, const uint32_t* which, const double* alpha_dev, double* g_part_out,
                                     double* diag_dev, double* dx_dev);
/* The HODLR counterpart of bgp_dense_loo_terms: the same outputs and errors, for the HODLR matrix K~ (not the dense K).
 * Always streamed, at every n, in the column slabs of bgp_hodlr_grad_terms (c columns, BGP_GRAD_CHUNK included):
 *   pass 1: per slab S = K~^-1 E_J by the row-restricted solve, d_j = S_jj for j in J;
 *   pass 2: beta by one solve, then per slab S again, its rows scaled by c, T = K~^-1 diag(c) S by a full c-column
 *           solve, and the contraction of beta_i alpha_j - T_ij over i in [0, n), j in J (every ordered pair, so this is
 *           the symmetrised A's sum) with diagA_j = alpha_j beta_j - T_jj.
 * Device workspace (doubles): n c + ceil(n / 32) P + ceil(n / 1024) (c / 32) P, plus 5 n + 64.  The sum order depends
 * only on n; where the solve has no atomics two identical calls return the same bits.  BGP_ERR_INVALID also on a
 * sharded factorisation (host-exchange shard or not), before anything is launched. */
int bgp_hodlr_loo_terms(bgp_hodlr_t* h, const uint32_t* which, const double* r, double* alpha_out, double* d_out,
                        double* beta_out, double* g_out, double* diag_out);
/* The HODLR counterpart of bgp_dense_predict (see there for the outputs, workspace and errors).
 * On a sharded factorisation with a matching communicator (see the multi-GPU block below) the call is COLLECTIVE, with
 * spec, xs and ns replicated: per test-point chunk each shard builds its own rows J of K(x, x*) into an N x c chunk, the
 * collective solve fills the other rows and runs the top levels, and the shard contracts over J
 * (bgp_hodlr_predict_local_dev's arithmetic, the prior on shard 0 only); one all-reduce of ns (VAR) or ns^2 (COV)
 * doubles adds the shards' parts, and every rank returns the same bits.  Everything is validated and reserved before
 * the first collective, and one all-reduce of a status value makes a failure on any rank an error on every rank.  The
 * number of chunks depends only on N, ns and BGP_PREDICT_CHUNK, which must therefore be the same on every rank.
 * Device workspace per shard (doubles), besides the result and xs, with nloc = the shard's rows:
 *   VAR  N*c + nloc*c + O(c)             COV  N*c + nloc*ns + split-K slices (c*ns each, at most 2^27; none with one)
 * A host-exchange shard returns BGP_ERR_INVALID, as before; it computes its part with bgp_hodlr_predict_local_dev. */
int bgp_hodlr_predict(bgp_hodlr_t* h, const bgp_kernel_spec_t* spec, const double* xs, int64_t ns, int32_t what,
                      double* out);
/* The HODLR counterpart of bgp_dense_predict_grad (see there).
 * On a sharded factorisation with a matching communicator the call is COLLECTIVE, as bgp_hodlr_predict is, with spec,
 * xs and ns replicated: per test-point chunk each shard builds its rows J of K(x, x*) into an N x c chunk, the
 * collective solve fills the other rows and runs the top levels, and the shard contracts var and dvar over J
 * (bgp_hodlr_predict_grad_local_dev's arithmetic, the prior on shard 0 only).  Two all-reduces end it: the ns doubles of
 * var, exactly as bgp_hodlr_predict issues it (so var is bgp_hodlr_predict's VAR output bit for bit on every rank), then
 * the ns * ndim of dvar.  Validation, reservation and the status all-reduce come before the first collective, as in
 * bgp_hodlr_predict.  Device workspace per shard (doubles), besides the results and xs: N*c + nloc*c + O(c * ndim).
 * A host-exchange shard returns BGP_ERR_INVALID; it computes its part with bgp_hodlr_predict_grad_local_dev. */
int bgp_hodlr_predict_grad(bgp_hodlr_t* h, const bgp_kernel_spec_t* spec, const double* xs, int64_t ns, double* var,
                           double* dvar);
/* One shard's part of the prediction: with J = this handle's own rows [row0, row0 + rows) ([0, N) unsharded),
 * B = K(x, x*) (N x ns) and P = B[J]^T W[J],
 *   VAR: out[ns]        = (add_prior ? k(x*_j, x*_j) : 0) - P_jj
 *   COV: out[i*ns + j]  = (add_prior ? K**(i,j) : 0) - P(i,j)     (row-major, bgp_hodlr_predict's orientation)
 * from w_dev, the full solved K^-1 B on the device (N x ns column-major, leading dimension ldw >= N; on a
 * host-exchange shard: solve_local_dev, the host's all-gather, solve_top_dev).  spec, xs and out as bgp_hodlr_predict.
 * Only rows J of w_dev are read, and only rows J of B are built (x is replicated on every shard).  The test points run
 * in bgp_hodlr_predict's chunks, so on an unsharded handle with add_prior = 1 the result is bit for bit what
 * bgp_hodlr_predict returns.  Summing the P shards' outputs, add_prior = 1 on exactly one of them, gives the prediction.
 * Issues no collective and works on any computed handle.  Workspace (doubles): VAR nloc*c + ns + O(c), COV nloc*ns +
 * ns^2 + split-K slices.  Errors, before anything is launched: BGP_ERR_NOT_COMPUTED before compute and on a shard whose
 * top levels are not finished; BGP_ERR_INVALID for an unknown `what`, ns < 0, a NULL w_dev with ns > 0 and ldw < N;
 * BGP_ERR_DIM when the spec's ndim differs from the handle's.  ns == 0 writes nothing. */
int bgp_hodlr_predict_local_dev(bgp_hodlr_t* h, const bgp_kernel_spec_t* spec, const double* xs, int64_t ns,
                                int32_t what, const double* w_dev, int64_t ldw, int32_t add_prior, double* out);
/* One shard's part of the variance gradient (GP.grad_predict): with J, B and w_dev as in bgp_hodlr_predict_local_dev,
 *   var[j]            = bgp_hodlr_predict_local_dev's VAR output for the same arguments, bit for bit
 *   dvar[j*ndim + q]  = (add_prior ? d k(x*_j, x*_j) / d x*_jq : 0) - 2 sum_{i in J} d k(x*_j, x_i) / d x*_jq W_ij
 * (dvar (ns x ndim) row-major, as bgp_hodlr_predict_grad).  Only rows J of w_dev are read, and only rows J of B are
 * built.  The chunks, contraction plan and evaluator are bgp_hodlr_predict_grad's, so on an unsharded handle with
 * add_prior = 1 and w_dev = apply_inverse's K^-1 B both outputs are its bits.  Summing the P shards' outputs, add_prior
 * = 1 on exactly one of them, gives var and dvar.  Issues no collective.  Workspace (doubles): the VAR part's plus
 * ns * ndim + O(c * ndim).  Errors: those of bgp_hodlr_predict_local_dev, and BGP_ERR_INVALID for ndim > BGP_MAX_DIM,
 * all before anything is launched.  ns == 0 writes nothing. */
int bgp_hodlr_predict_grad_local_dev(bgp_hodlr_t* h, const bgp_kernel_spec_t* spec, const double* xs, int64_t ns,
                                     const double* w_dev, int64_t ldw, int32_t add_prior, double* var, double* dvar);

/* ------------------------------------------------------------------------------------------
 * Draws from N(mean, C) on the device: GP.sample_conditional / GP.sample with a caller's random generator (the
 * reference draws with numpy's multivariate_normal, an SVD of C on the host: utils.py:19-33, gp.py:547-599).
 *   A   = sym(C) + jitter * I, sym(C) the LOWER triangle C[i*ns + j], i >= j, of the row-major C, mirrored
 *   L   = the lower Cholesky factor of A (bgp_dense_compute's blocked Cholesky)
 *   out[a*ns + j] = mean[j] + sum_{i <= j} z[a*ns + i] L(j, i)     (size x ns row-major: draws = mean + z L^T)
 * mean (ns) and z (size x ns row-major, the caller's standard normals) are host arrays.  Fewer than
 * BGP_SAMPLE_DMMA_ROWS draws run as one row of threads per draw (bgp_dense_apply_sqrt's arithmetic plus the mean: each
 * draw reads L once); more run as a triangular GEMM on the DMMA pipe, one descriptor per 128 columns of out, its K
 * stopping at the tile's last column.  Both add in a fixed order (no atomics): identical inputs give identical bits.
 * bgp_mvn_sample takes C from the host.  bgp_dense_sample and bgp_hodlr_sample build C on the device exactly as the
 * COV branch of bgp_dense_predict / bgp_hodlr_predict does (spec, xs, ns as there) and C never leaves the device, so
 * bgp_dense_sample equals bgp_mvn_sample on bgp_dense_predict's output bit for bit; for HODLR the same holds wherever its
 * predict is reproducible (N <= 1024, see bgp_dense_predict).
 * Workspace (doubles): ns^2 (C, factorised in place) + (2 size + 1) ns, on top of the predict's for the fused entries.
 * Errors: BGP_ERR_NOT_COMPUTED before compute and on a dense handle restored by bgp_dense_import_factor; BGP_ERR_DIM
 * when the spec's ndim differs from the handle's; BGP_ERR_INVALID for ns < 0, size < 0, a negative or non-finite
 * jitter and on any sharded HODLR handle (the sharded solver samples through bgp_mvn_sample on its collective
 * prediction); BGP_ERR_NOMEM when the workspace cannot be allocated; BGP_ERR_LINALG, "k-th leading minor of the array
 * is not positive definite", when A is not (a negative predictive variance, a NaN, a singular C with jitter 0).  The
 * solver's handle is unchanged by any outcome.  ns == 0 or size == 0 writes nothing.
 * ------------------------------------------------------------------------------------------ */
/* Draws from which the product runs on the DMMA pipe.  On one H100 (700 W) the row path takes 0.05 / 0.13 ms for 1-7
 * draws at ns = 256 / 1024 against 0.08 / 0.20 ms for the DMMA path, and loses at ns >= 4096 (0.82-0.90 vs 0.70 ms);
 * tools/sample_bench.py, DESIGN.md §6. */
#define BGP_SAMPLE_DMMA_ROWS 8
int bgp_mvn_sample(const double* cov, int64_t ns, const double* mean, const double* z, int64_t size, double jitter,
                   double* out);
int bgp_dense_sample(bgp_dense_t* h, const bgp_kernel_spec_t* spec, const double* xs, int64_t ns, const double* mean,
                     const double* z, int64_t size, double jitter, double* out);
int bgp_hodlr_sample(bgp_hodlr_t* h, const bgp_kernel_spec_t* spec, const double* xs, int64_t ns, const double* mean,
                     const double* z, int64_t size, double jitter, double* out);
/* device-event timing (ms) of the calling thread's last successful sampling call: [0] the covariance (its build on
 * the device for the fused entries, its upload for bgp_mvn_sample) and the upload of mean and z, [1] symmetrisation +
 * Cholesky, [2] the product. */
int bgp_sample_last_timing(double* ms3);

/* Symmetric factor of a computed (unsharded) HODLR matrix, K~ = W W^T (Ambikasaran, O'Neil & Singh, arXiv:1405.0223):
 * W = W_leaf W_{k-1} ... W_0, W_leaf = blockdiag(L D^1/2) of the leaves' L D L^T, and W_l block diagonal over the
 * nodes of level l with blocks I + Q X Q^T (Q orthonormal, from the node's ACA factors).  Built on the device from what
 * compute() leaves there, on the first of these calls after a compute(), and kept until the next compute(); compute()
 * and every other entry point do no work for it.  Deterministic: the same factorisation gives the same bits.
 * Each node's bases come from equilibrated shifted CholeskyQR3, or, where those miss |Q^T Q - I| <= 1e-13 or the Gram
 * matrix has no Cholesky factor (numerically dependent ACA columns, e.g. a block the ACA returned dense), from
 * Householder QR: every positive-definite K~ with finite factors is factored.
 * Device memory, kept on the handle: N * (sum_l r_l + max_l r_l + 64) doubles (the factor panel, the copy of one
 * level's columns, the apply's 64-column staging), 8 (2r)^2 + 6 r^2 doubles per node, and the products' workspace.
 * Limits: a level's rank r at most 2048 (each node's 2r x 2r Cholesky and its Householder QR run in one CTA, whose
 * time grows as r^3); levels of any width (the level kernels launch in slabs of 32767 nodes).
 * Diagnostic: BGP_SYM_QR=householder (read when the factor is built) sends every node of nonzero rank through the
 * Householder QR instead of CholeskyQR3; the two give the same W to rounding.
 * Errors: BGP_ERR_NOT_COMPUTED; BGP_ERR_INVALID on a host-exchange shard (checked first; see the sharded entry points
 * below) and, before anything is launched, for a node whose level rank is above the limit (naming the node, its rank
 * and the limit); BGP_ERR_LINALG when K~ is not positive definite, naming the leaf and row (a pivot D_ii that is not a
 * finite positive number) or the node whose 2r x 2r step I + M = L L^T has no Cholesky factor, and when a node's
 * factors are not finite.
 * Sharded (opts.shard_count > 1, DESIGN.md §5): on a shard with a matching communicator these three calls are
 * COLLECTIVE.  The factor splits at the shard cut: each shard factors its leaves and owned levels on its own rows
 * (each owned node also updating the top levels' columns there), one all-gather of its rows of those columns, then the
 * nodes above the cut on every shard; log|K~| is one all-reduce of the shards' partial sums.  Every check and
 * reservation runs before an all-reduce of a status, and the local build ends with a second one before the all-gather:
 * a shard whose leaf or node has no factor returns BGP_ERR_LINALG naming it, and every other shard BGP_ERR_LINALG naming
 * that shard.  bgp_hodlr_sym_apply takes z replicated on every shard and returns the result replicated (W: the top
 * levels, this shard's levels and leaves on its rows, an all-gather of the rows; W^T the reverse).  After any failure
 * the factor is not current and the handle stays usable.
 * Device memory per shard, kept on the handle: N * (R_top + 64) + nloc * R_loc doubles (the top part of the factor
 * panel, the apply's staging, the local part), the copy of one level's columns (N or nloc rows), the per-node blocks of
 * the shard's nodes and the nodes above the cut, the products' workspace, and the all-gather's staging
 * (P + 1) * max(R_top, 64) * rows_pad doubles; R_top and R_loc are the column counts of the top and local U panels. */
int bgp_hodlr_sym_factor(bgp_hodlr_t* h);
/* z (n x nrhs, column-major, leading dimension ldz, host) <- W z (transpose = 0) or W^T z, in place.  With z standard
 * normal, W z is distributed as N(0, K~). */
int bgp_hodlr_sym_apply(bgp_hodlr_t* h, double* z, int64_t nrhs, int64_t ldz, int32_t transpose);
/* log|K~| = sum log D_ii + 2 sum_v log|det(I + X_v)|: an independent evaluation of bgp_hodlr_log_determinant's value. */
int bgp_hodlr_sym_log_determinant(bgp_hodlr_t* h, double* out);
/* The symmetric factor on a host-exchange shard, step by step (the order of export_top / import_top / finish_top /
 * solve_{local,top}_dev below; the host runs the all-gather):
 *   1. bgp_hodlr_sym_factor_local on every shard, after its factorisation is finished (bgp_hodlr_finish_top): the
 *      leaves, the owned levels and this shard's rows of the top levels' columns.  Rebuilds from scratch when called
 *      again.  Errors as bgp_hodlr_sym_factor's, naming this shard's leaf or node.
 *   2. bgp_hodlr_sym_export_top into the shard's slot of a (P, cols, rows_pad) device buffer (export_top's layout; cols
 *      = bgp_hodlr_top_panel's cols), the host all-gathers it, bgp_hodlr_sym_import_top on every shard.
 *   3. bgp_hodlr_sym_finish_top on every shard, once: the nodes above the cut; marks the factor current and returns
 *      this shard's PARTIAL log|K~| (its leaves and owned nodes, plus the nodes above the cut on shard 0 only), whose
 *      sum over the shards is log|K~|.  It is also what bgp_hodlr_sym_log_determinant would hold.
 *   4. bgp_hodlr_sym_apply_local_dev / bgp_hodlr_sym_apply_top_dev, in place on an (N x nrhs) column-major device block
 *      with ldz >= N, z replicated: W z is top, then local, then the host assembles rows [row0_s, row0_s + rows_s)
 *      from shard s; W^T z is local, the host assembles the rows and copies them to every shard, then top.  The local
 *      part reads and writes this shard's rows only.
 * On an unsharded handle the local part is the whole factor and the top part does nothing (export / import copy
 * nothing), and the apply entries build the factor on first use; local + top give bgp_hodlr_sym_apply's bits and the
 * partial log|K~| is bgp_hodlr_sym_log_determinant's value.  Call-order errors, returned before anything is launched:
 * BGP_ERR_NOT_COMPUTED for factor_local before the factorisation is finished, for export / import / finish before
 * factor_local or after it failed, and for the apply entries on a shard before finish; BGP_ERR_INVALID for export /
 * import / finish once the factor is complete (a second finish) and for a rows_pad below this shard's rows (export) or
 * the largest shard's rows (import).  Issue no collective. */
int bgp_hodlr_sym_factor_local(bgp_hodlr_t* h);
int bgp_hodlr_sym_export_top(bgp_hodlr_t* h, double* buf_dev, int64_t rows_pad);
int bgp_hodlr_sym_import_top(bgp_hodlr_t* h, const double* all_buf_dev, int64_t rows_pad);
int bgp_hodlr_sym_finish_top(bgp_hodlr_t* h, double* partial_logdet);
int bgp_hodlr_sym_apply_local_dev(bgp_hodlr_t* h, double* z_dev, int64_t nrhs, int64_t ldz, int32_t transpose);
int bgp_hodlr_sym_apply_top_dev(bgp_hodlr_t* h, double* z_dev, int64_t nrhs, int64_t ldz, int32_t transpose);
/* Test diagnostic: max over the nodes and halves of max |Q^T Q - I| of the symmetric factor's orthonormal bases. */
int bgp_selftest_hodlr_sym_orthogonality(bgp_hodlr_t* h, double* out);
/* Test diagnostic: how many nodes of each level (0 = the root) the last symmetric-factor build orthonormalised by
 * Householder QR rather than CholeskyQR3.  counts[l] for l < min(cap, *nlev); *nlev = the number of internal levels. */
int bgp_selftest_hodlr_sym_householder_nodes(bgp_hodlr_t* h, int32_t* counts, int32_t cap, int32_t* nlev);
/* Device-event time (ms) of the last symmetric-factor build ([0]) and of the last bgp_hodlr_sym_apply's products
 * ([1]: summed over its 64-column groups, host transfers excluded); 0 before the first. */
int bgp_hodlr_sym_last_timing(const bgp_hodlr_t* h, double* ms2);

/* Tree / index structure introspection (bit-exact parity target; hodlr.h:48-61).
 * Nodes are listed in the reference's PRE-ORDER construction order. */
typedef struct bgp_hodlr_node_info {
  int32_t start, size, half; /* half = size/2 (hodlr.h:48); children are [start,half) and [start+half,size-half) */
  int32_t is_leaf;
  int32_t parent;            /* pre-order index of the parent, -1 for the root                     */
  int32_t direction;         /* 0 = left child, 1 = right child (hodlr.h:58-61)                    */
  int32_t depth;
  int32_t rank;              /* ACA rank of the node's off-diagonal block (0 for leaves)           */
  int32_t rng_draws;         /* number of mt19937 words the node's ACA consumed                    */
  int32_t dense_fallback;    /* 1 if the rows ran out and the dense factorisation was returned (hodlr.h:161-176) */
} bgp_hodlr_node_info_t;
int bgp_hodlr_num_nodes(const bgp_hodlr_t* h, int64_t* out);
int bgp_hodlr_node_info(const bgp_hodlr_t* h, bgp_hodlr_node_info_t* out /* num_nodes */);
/* ACA pivots of node `node` (pre-order index): rows[k], cols[k] for k < rank, block-relative. */
int bgp_hodlr_node_pivots(const bgp_hodlr_t* h, int64_t node, int32_t* rows, int32_t* cols);
/* Diagnostics: the low-rank factors of internal node `node` as the ACA left them (they are not modified afterwards).
 * out: host buffer (size x rank, column-major, ld size; size and rank from bgp_hodlr_node_info).  Rows [0, half) hold
 * V_[0] (normalised residual rows, indexed by the left half's columns), rows [half, size) hold U_[1] (residual columns,
 * indexed by the right half's rows), so the block K[right, left] ~ out[half:, :] out[:half, :]^T.  A dense-fallback node
 * (exhaust_mode = DENSE) holds V = I and U = the block itself.  Nothing is written for rank 0.  Single-GPU only:
 * BGP_ERR_INVALID on a sharded factorisation; BGP_ERR_INDEX for a leaf or an out-of-range node; BGP_ERR_NOT_COMPUTED
 * before compute. */
int bgp_hodlr_node_factors(const bgp_hodlr_t* h, int64_t node, double* out);
/* Diagnostics: how often the per-node-stream ACA of the last compute left the common path of its speculative row draws
 * (csrc/hodlr_aca2.cuh).  out4 = [0] Lemire rejections redone inside a batch, [1] batches truncated before a rejecting
 * last draw, [2] rejecting draws of one-candidate batches drawn sequentially, [3] commits that replayed the mt19937
 * stream to the winning draw instead of taking the saved end-of-batch state.  All zero for rng_mode = REFERENCE, which
 * draws one row at a time.  BGP_ERR_NOT_COMPUTED before compute. */
int bgp_hodlr_last_draw_paths(const bgp_hodlr_t* h, uint64_t* out4);
/* Diagnostics: the work units of the per-node-stream ACA's candidate evaluation in the last compute
 * (csrc/hodlr_aca2.cuh, a2_eval_kernel; one unit = one candidate block against 128 columns of the block).
 * out2 = [0] units pulled by the evaluation kernel, [1] units in which at least one candidate survived the
 * 128-column bound and was evaluated (all of [0] that have columns when bound culling is off).  Decisions never
 * depend on these counts.  All zero for rng_mode = REFERENCE.  BGP_ERR_NOT_COMPUTED before compute. */
int bgp_hodlr_last_eval_units(const bgp_hodlr_t* h, uint64_t* out2);
/* Device-event timings of the last compute, ms: [0] leaves (build+factor; stream A, CONCURRENT with [1]),
 * [1] ACA (stream B, from the start of compute), [2] up-sweep (panel finalisation + leaf solves + level sweeps, from the
 * moment both streams have drained), [3] total compute, [4] last solve.  [3] ~ max([0], [1]) + host gap + [2]. */
int bgp_hodlr_last_timing(const bgp_hodlr_t* h, double* ms5);
/* The last bgp_hodlr_grad_terms[_local_dev]: out4 = [0] ms in the solves (alpha and K^-1), [1] ms in the contraction (with the
 * diagonal and the reductions), both measured with CUDA events only while profiling is on (bgp_hodlr_set_profiling;
 * every K^-1 slab then waits for its events) and 0 otherwise, [2] number of K^-1 slabs, [3] columns per slab ([2] and
 * [3] are 0 on the resident path). */
int bgp_hodlr_last_grad_timing(const bgp_hodlr_t* h, double* out4);
/* Algorithmic work of the last compute (SURVEY.md §8d): [0] kernel evaluations, [1] bytes, [2] flops,
 * [3] sum of per-level max ranks R, [4] leaf size m, [5] number of levels. */
int bgp_hodlr_last_work(const bgp_hodlr_t* h, double* w6);
/* Optional per-kernel timing of the lock-step ACA loop: with profiling on, every launch is bracketed by CUDA events on
 * its stream.  p12 = [0] summed a2_eval launch time ms, [1] launches of each kernel (= lock-step iterations),
 * [2] candidate-row entries verified against the 1e-14 pivot threshold (hodlr.h:191), [3] residual-update FMAs,
 * [4] candidate rows examined, [5] entries of [2] that were actually evaluated (the others were bounded below the
 * threshold from the kernel's decay and the factor magnitudes, without evaluation; decisions are identical),
 * [6..11] summed launch times ms of a2_eval (+ its all-reduce when sharded), a2_decide, a2_vrow, a2_pivot,
 * a2_vnorm_ucol, a2_finish. */
int bgp_hodlr_set_profiling(bgp_hodlr_t* h, int on);
int bgp_hodlr_last_aca_profile(const bgp_hodlr_t* h, double* p12);

/* Diagnostics: the dense building blocks of the big-rank Woodbury step (csrc/hodlr_lu.cuh, csrc/gemm_dmma.cuh),
 * callable on their own with HOST pointers so the tests can check them against LAPACK.
 *   bgp_selftest_lu: S (n x n, column-major) is LU-factored with partial pivoting in blocks of 32, R (n x nrhs,
 *     column-major, ld n) is overwritten by S^-1 R, *logdet = log|det S|      (stands in for Eigen::FullPivLU,
 *     hodlr.h:228-234, :90-93, :250).
 *   bgp_selftest_gemm: C (m x n, column-major ldc) -= A' B'; A' (m,k) = a_kcontig ? A[m*lda+k] : A[k*lda+m];
 *     B' (k,n) = b_kcontig ? B[n*ldb+k] : B[k*ldb+n].  All four (a_kcontig, b_kcontig) variants are built: (0,0) is the
 *     one the dense Cholesky's trailing updates use, (1,0) the Fisher rows' second product.  mode: bit 0 (1) C += A'B'
 *     with atomics instead, bit 8 (256) only entries with row >= column are written (the Cholesky's lower-triangular
 *     output). */
int bgp_selftest_lu(int32_t n, int32_t nrhs, const double* S_host, double* R_host, double* logdet);
int bgp_selftest_gemm(int32_t a_kcontig, int32_t b_kcontig, int32_t m, int32_t n, int32_t k, const double* A_host,
                      int64_t lda, const double* B_host, int64_t ldb, double* C_host, int64_t ldc, int32_t mode);

/* Multi-GPU (SURVEY.md §8e).  With a communicator (bgp_comm_init) whose size and rank match opts.shard_count /
 * opts.shard_rank, bgp_hodlr_compute[_dev] is COLLECTIVE and complete: local sub-tree, all-gather of the rows this shard
 * owns of the top-level factor panel (pack kernel -> ncclAllGather -> unpack kernels on the solver's stream), the nodes
 * above the cut, log-det all-reduce; apply_inverse / dot_solve are collective too (replicated right-hand side, one
 * all-gather of the locally solved slices), and so are grad_terms and predict.  WITHOUT a communicator (a "host-exchange shard": no communicator, or one
 * whose size or rank does not match) the same steps are exposed one by one so that a host can run the exchange itself.
 * The P shards may be P processes or P handles in one process, on any devices.  The call order is:
 *   1. bgp_hodlr_compute[_dev] on every shard (opts.shard_rank = s, opts.shard_count = P, rng_mode = per-node).  It
 *      returns with the local sub-tree factored and applied to this shard's rows of the top panel; the handle is not
 *      computed yet (bgp_hodlr_computed = 0, solves return BGP_ERR_NOT_COMPUTED).
 *   2. bgp_hodlr_export_top on every shard into its slot of a (P, cols, rows_pad) buffer, rows_pad >= the largest
 *      bgp_hodlr_shard_rows; the host all-gathers the buffer (every device stream involved must have finished).
 *   3. bgp_hodlr_import_top on every shard; the top panels of all shards are then identical.
 *   4. bgp_hodlr_finish_top on every shard, exactly once.
 *   5. solves: bgp_hodlr_solve_local_dev on every shard with the same right-hand side, the host assembles rows
 *      [row0_s, row0_s + rows_s) from shard s and copies the assembled block to every shard, then
 *      bgp_hodlr_solve_top_dev on every shard; every shard then holds the whole solution.
 * The full solves (bgp_hodlr_apply_inverse, bgp_hodlr_dot_solve[_dev], bgp_hodlr_get_inverse), like grad_terms,
 * predict and node_factors, return BGP_ERR_INVALID on a host-exchange shard: they need the other shards' rows.  The
 * gradient runs there as bgp_hodlr_grad_terms_local_dev on every shard with the solved alpha, the host summing g and
 * assembling the diag slices; with a matching communicator bgp_hodlr_grad_terms does all of it collectively.  The
 * prediction runs there as bgp_hodlr_predict_local_dev on every shard with the solved K^-1 K(x, x*), the host summing
 * the outputs (the prior on one shard); with a matching communicator bgp_hodlr_predict does it collectively.  The
 * variance gradient likewise runs as bgp_hodlr_predict_grad_local_dev, or collectively as bgp_hodlr_predict_grad.
 * bgp_hodlr_log_determinant on a host-exchange shard returns that shard's PARTIAL log-determinant: its own leaves and
 * sub-tree nodes, plus the nodes above the cut on shard 0 only, so the sum over the P shards is log det K.
 *   bgp_hodlr_top_panel(h, &ptr_dev, &row0, &rows, &cols, &ld): device pointer to the (N x cols) column-major panel of
 *     the levels above the cut (ld = N), and this shard's rows [row0, row0 + rows).                               */
int bgp_hodlr_top_panel(bgp_hodlr_t* h, double** ptr_dev, int64_t* row0, int64_t* rows, int64_t* cols, int64_t* ld);
/* pack this shard's rows of the top panel into a contiguous (cols x rows_pad) device buffer (column c at c*rows_pad),
 * and scatter the all-gathered buffers (shard s at s*cols*rows_pad) of all shards back into the panel.  Both are valid
 * only between step 1 and step 4: BGP_ERR_NOT_COMPUTED before any compute, BGP_ERR_INVALID on an unsharded or already
 * finished factorisation.  BGP_ERR_INVALID also when rows_pad is smaller than this shard's rows (export) or than the
 * largest shard's rows (import), also when the panel has no columns (a rank-0 top: nothing is copied). */
int bgp_hodlr_export_top(bgp_hodlr_t* h, double* buf_dev, int64_t rows_pad);
int bgp_hodlr_import_top(bgp_hodlr_t* h, const double* all_buf_dev, int64_t rows_pad);
/* row range [row0, row0+rows) owned by shard `s` (same on every shard).  BGP_ERR_INDEX if `s` is out of range, and for
 * every `s` when the last compute was unsharded or failed because the tree cannot be cut shard_count ways. */
int bgp_hodlr_shard_rows(const bgp_hodlr_t* h, int32_t s, int64_t* row0, int64_t* rows);
/* Gram/LU/log-det/update of the nodes above the shard cut, on the imported top panel; marks the handle computed.  Once
 * per compute: BGP_ERR_NOT_COMPUTED before any compute, BGP_ERR_INVALID on an unsharded factorisation or a second call. */
int bgp_hodlr_finish_top(bgp_hodlr_t* h);
/* The library's NCCL communicator (one per process).  Rank 0 makes a unique id (128 bytes), the host broadcasts it over
 * whatever it has (torch.distributed, MPI, a file), every rank calls bgp_comm_init.  `nccl_path` may be NULL: the library
 * already loaded in the process (torch's libnccl.so.2) is used, else libnccl.so.2 is dlopen'ed. */
int bgp_comm_unique_id(void* out128, const char* nccl_path);
int bgp_comm_init(const void* id128, int rank, int world, const char* nccl_path);
int bgp_comm_destroy(void);
int bgp_comm_size(void);
/* sharded solve (step 5 above): local part, then (host all-gathers the vector), then top part, in place on an
 * (N x nrhs) column-major device block with ldb >= N.  BGP_ERR_NOT_COMPUTED before finish_top. */
int bgp_hodlr_solve_local_dev(bgp_hodlr_t* h, double* b_dev, int64_t nrhs, int64_t ldb);
int bgp_hodlr_solve_top_dev(bgp_hodlr_t* h, double* b_dev, int64_t nrhs, int64_t ldb);

/* ------------------------------------------------------------------------------------------
 * Device memory helpers so a host without torch can stage inputs (bench "value" leg).
 * ------------------------------------------------------------------------------------------ */
int bgp_dev_alloc(void** ptr_dev, size_t bytes);
int bgp_dev_free(void* ptr_dev);
/* bgp_dev_upload returns once the data is on the device (also from pageable host memory), so any library call made
 * after it, on whichever of the library's streams, reads the uploaded bytes. */
int bgp_dev_upload(void* dst_dev, const void* src_host, size_t bytes);
int bgp_dev_download(void* dst_host, const void* src_dev, size_t bytes);
int bgp_dev_synchronize(void);
int bgp_host_alloc_pinned(void** ptr, size_t bytes);
int bgp_host_free_pinned(void* ptr);

#ifdef __cplusplus
}
#endif
#endif /* BGP_B200_H_ */
