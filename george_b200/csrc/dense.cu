// dense.cu — K3: dense solver behind BasicSolver (replaces src/george/solvers/basic.py:51-121, i.e.
// kernel.get_value + scipy.linalg.cholesky / cho_solve, LAPACK dpotrf/dpotrs).
//
// The covariance matrix is generated on the device by the fused kernel-matrix build (kmat.cu) with yerr^2 already on
// the diagonal, factorised in place (blocked right-looking Cholesky, lower factor L with K = L L^T; the reference keeps
// the upper factor U = L^T, basic.py:68) and never leaves HBM.  log-det = 2 sum log L_ii (basic.py:69).
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <vector>

#include "common.cuh"
#include "gemm_dmma.cuh"
#include "kernel_eval.cuh"
#include "linalg.cuh"

namespace bgp {
int upload_program(const DevProgram& P, DevBuf<DevProgram>& buf, cudaStream_t s);
int kmat_symmetric_launch(const DevProgram* dprog, int nd, const double* x, int64_t n, const double* diag_add,
                          double* out, int64_t ld, cudaStream_t s);
int kmat_symmetric_launch_auto(const DevProgram& P, const DevProgram* dprog, const double* x, int64_t n,
                               const double* diag_add, double* out, int64_t ld, cudaStream_t s);
int kmat_grad_contract_launch(const DevProgram* dprog, int nd, int np, const unsigned* which_dev, const double* x,
                              int64_t n, const double* M, int64_t ldm, const double* alpha, double ca, double cm,
                              double* g_dev, double* diag_dev, DevBuf<double>& scratch, cudaStream_t s);
int kmat_grad_contract_members(const DevProgram* dprogs, int np, const unsigned* which_dev, const double* x, int64_t n,
                               const double* M, int64_t ldm, int64_t mstride, const double* alpha, int64_t astride,
                               double ca, double cm, double* g_dev, int64_t gstride, double* diag_dev, int64_t dstride,
                               int members, DevBuf<double>& scratch, cudaStream_t s);
int fill_identity_launch(double* A, int64_t n, cudaStream_t s);
int grad_x_resident_launch(const DevProgram& P, const DevProgram* dprog, const double* x, int64_t n, double* Kinv,
                           const double* alpha, double* dx_dev, DevBuf<double>& scratch, cudaStream_t s);
int loo_weights_launch(const double* alpha, const double* d, int64_t n, double* q, double* c, cudaStream_t s);
int scale_rows_launch(double* X, int64_t n, int64_t ncols, int64_t ldx, const double* w, bool sqrt_w, cudaStream_t s);
int slab_diag_launch(const double* W, int64_t ldw, int64_t j0, int64_t nc, double* d, cudaStream_t s);
int loo_check_diag(const double* d, int64_t n);
int loo_weights_members(const double* alpha, const double* d, int64_t n, double* q, double* c, int members,
                        cudaStream_t s);
int scale_rows_members(double* X, int64_t n, int64_t ncols, int64_t ldx, const double* w, bool sqrt_w, int members,
                       int64_t xstride, int64_t wstride, cudaStream_t s);
int slab_diag_members(const double* W, int64_t ldw, int64_t j0, int64_t nc, double* d, int members, int64_t wstride,
                      int64_t dstride, cudaStream_t s);
int fill_identity_members(double* A, int64_t n, int members, cudaStream_t s);
int kmat_general_launch_auto(const DevProgram& P, const DevProgram* dprog, const double* x1, int64_t n1, const double* x2,
                             int64_t n2, double* out, int64_t ld, cudaStream_t s);
int kmat_diagonal_launch(const DevProgram* dprog, const double* x1, const double* x2, int64_t n, double* out,
                         cudaStream_t s, int members = 1, int64_t ostride = 0);
int kmat_symmetric_batch_launch_auto(const DevProgram* P, const DevProgram* dprogs, int B, const double* x, int64_t n,
                                     const double* diag_add, double* out, int64_t mstride, DevBuf<double>& scratch,
                                     cudaStream_t s);
int kmat_general_batch_launch_auto(const DevProgram* P, const DevProgram* dprogs, int B, const double* x1, int64_t n1,
                                   const double* x2, int64_t n2, double* out, int64_t ld, int64_t mstride,
                                   DevBuf<double>& scratch, cudaStream_t s);
int kmat_matvec_batch_launch(const DevProgram* dprogs, int nd, int members, const double* x1, int64_t n1,
                             const double* x2, int64_t n2, const double* V, int64_t vstride, double* out,
                             int64_t ostride, double* partial, cudaStream_t s);
int64_t matvec_partial_size(int64_t n1, int64_t n2);
int64_t predict_chunk_cols(int64_t n, int64_t multiple);
int64_t predict_var_partial_size(int64_t n, int64_t c);
int predict_var_batch_launch(const double* B, int64_t ldb, const double* W, int64_t ldw, int64_t n, int64_t c,
                             const double* kdiag, double* var, int members, int64_t mstride, int64_t vstride,
                             DevBuf<double>& scratch, cudaStream_t s);
void predict_gemm_plan(int64_t m, int64_t nn, int64_t K, int64_t* nsplit_out, int64_t* klen_out);
int predict_gemm_sub_members(const double* A, int64_t lda, const double* B, int64_t ldb, int64_t m, int64_t nn,
                             int64_t K, bool lower, double* C, int64_t ldc, int members, int64_t abstride,
                             int64_t cstride, DevBuf<double>& slices, DevBuf<GemmDesc>& descs, cudaStream_t s);
int kmat_x1_grad_matvec_launch(const DevProgram& P, const DevProgram* dprog, const double* x1, int64_t n1,
                               const double* x2, int64_t n2, const double* V, int64_t ldv, double scale, int add_prior,
                               double* out, DevBuf<double>& scratch, cudaStream_t s);
int kmat_x1_grad_matvec_members(const DevProgram* P, const DevProgram* dprogs, int members, const double* x1,
                                int64_t n1, const double* x2, int64_t n2, const double* V, int64_t ldv,
                                int64_t vstride, double scale, int add_prior, double* out, int64_t ostride,
                                DevBuf<double>& scratch, cudaStream_t s);
int64_t x1_grad_partial_size(int64_t n1, int64_t n2, int nd);
int predict_var_launch(const double* B, int64_t ldb, const double* W, int64_t ldw, int64_t n, int64_t c,
                       const double* kdiag, double* var, DevBuf<double>& scratch, cudaStream_t s);
int predict_gemm_sub(const double* A, int64_t lda, const double* B, int64_t ldb, int64_t m, int64_t nn, int64_t K,
                     bool lower, double* C, int64_t ldc, DevBuf<double>& slices, DevBuf<GemmDesc>& descs, cudaStream_t s);
int predict_gemm_sub_bt(const double* A, int64_t lda, const double* B, int64_t ldb, int64_t m, int64_t nn, int64_t K,
                        bool lower, double* C, int64_t ldc, DevBuf<double>& slices, DevBuf<GemmDesc>& descs,
                        cudaStream_t s);
int predict_gemm_sub_bt_members(const double* A, int64_t lda, const double* B, int64_t ldb, int64_t m, int64_t nn,
                                int64_t K, bool lower, double* C, int64_t ldc, int members, int64_t abstride,
                                int64_t cstride, DevBuf<double>& slices, DevBuf<GemmDesc>& descs, cudaStream_t s);
int kmat_gradient_plane_launch(const DevProgram* dprog, int np, int p, const double* x, int64_t n, double* out,
                               int64_t ldo, cudaStream_t s);
int kmat_gradient_plane_members(const DevProgram* dprogs, int np, int p, const double* x, int64_t n, double* out,
                                int64_t ldo, int64_t ostride, int members, cudaStream_t s);

constexpr int DN_NB = 64;   // inner panel width (diagonal block in shared memory)
constexpr int DN_MB = 256;  // middle block of the delayed-update hierarchy (see dense_potrf)
constexpr int DN_OB = 2048; // outer block: trailing updates beyond it run with K = 2048 on the tensor pipe (config 4,
                            // N = 32768, on H100 at 400 W: potrf 540 ms; BGP_DENSE_OB selects other widths for a sweep)

// ---- diagonal block Cholesky (NB x NB): one thread per ROW, the row lives in registers ------------------------------
// Right-looking, fully unrolled: at step k every thread scales its entry of column k and applies the rank-1 update to
// its own row; the only exchanges are the pivot and the scaled column, through (double-buffered) shared memory, two
// barriers per step.  info != 0 when a pivot is not positive (LAPACK dpotrf's info = k+1; scipy raises LinAlgError).
// Batched factorisations (bgp_dense_batch_*) run member blockIdx.y on the slab A + blockIdx.y * mstride with its own
// info word; a single factorisation launches one member.
__global__ void __launch_bounds__(DN_NB) potf2_kernel(double* __restrict__ A, int64_t lda, int nb, int* info, int k0,
                                                      int64_t mstride) {
  A += blockIdx.y * mstride;
  info += blockIdx.y;
  __shared__ double col[2][DN_NB];
  __shared__ double piv[2];
  const int i = threadIdx.x;
  double a[DN_NB];
#pragma unroll
  for (int j = 0; j < DN_NB; ++j) a[j] = (i < nb && j < nb) ? A[(int64_t)j * lda + i] : (i == j ? 1.0 : 0.0);
  if (i == 0) piv[0] = a[0];
  __syncthreads();
#pragma unroll
  for (int k = 0; k < DN_NB; ++k) {
    const double d = piv[k & 1];
    if (!(d > 0.0)) {  // also catches NaN; uniform: every thread reads the same pivot
      if (i == 0) atomicCAS(info, 0, k0 + k + 1);
      return;
    }
    // 1/sqrt(d) (one MUFU + Newton steps) instead of sqrt followed by a division: this scalar chain is the critical
    // path of the whole factorisation step; the factor entries differ from sqrt/divide by <= 2 ulp
    const double rinv = rsqrt(d);
    const double lik = (i == k) ? d * rinv : a[k] * rinv;
    a[k] = lik;
    col[k & 1][i] = lik;
    __syncthreads();
#pragma unroll
    for (int j = k + 1; j < DN_NB; ++j) a[j] = fma(-lik, col[k & 1][j], a[j]);  // entries above the diagonal are scratch
    if (k + 1 < DN_NB) {
      if (i == k + 1) piv[(k + 1) & 1] = a[k + 1];
      __syncthreads();
    }
  }
  if (i < nb) {
#pragma unroll
    for (int j = 0; j < DN_NB; ++j)
      if (j < nb) A[(int64_t)j * lda + i] = (j <= i) ? a[j] : 0.0;  // explicit zeros above the diagonal of the block
  }
}

// ---- panel solve: rows below the diagonal block, L21 = A21 * L11^-T; one row per thread ---------------------------
// Column-oriented substitution (x_j = w_j / l_jj, then w_q -= x_j l_qj for q > j): the 2016 updates of a row are
// independent FMAs instead of 64 dependent dot products; the 64 divisions are multiplications by reciprocals computed
// once per CTA.
// (member blockIdx.y of a batch: slab A + blockIdx.y * mstride, info word info[blockIdx.y])
__global__ void __launch_bounds__(128, 1) trsm_panel_kernel(double* __restrict__ A, int64_t lda, int64_t rows, int nb,
                                                         const int* info, int64_t mstride) {
  __shared__ double l[DN_NB][DN_NB + 1];
  __shared__ double rl[DN_NB];
  A += blockIdx.y * mstride;
  if (info[blockIdx.y] != 0) return;
  for (int t = threadIdx.x; t < DN_NB * DN_NB; t += blockDim.x) {
    const int i = t % DN_NB, j = t / DN_NB;
    l[i][j] = (i < nb && j < nb) ? A[(int64_t)j * lda + i] : (i == j ? 1.0 : 0.0);
  }
  __syncthreads();
  if (threadIdx.x < DN_NB) rl[threadIdx.x] = 1.0 / l[threadIdx.x][threadIdx.x];
  __syncthreads();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows) return;
  double* row = A + nb + i;  // element (nb + i, j) at row[j*lda]
  double w[DN_NB];
#pragma unroll
  for (int j = 0; j < DN_NB; ++j) w[j] = (j < nb) ? row[(int64_t)j * lda] : 0.0;
#pragma unroll
  for (int j = 0; j < DN_NB; ++j) {
    const double xj = w[j] * rl[j];
    w[j] = xj;
#pragma unroll
    for (int q = j + 1; q < DN_NB; ++q) w[q] = fma(-xj, l[q][j], w[q]);
  }
#pragma unroll
  for (int j = 0; j < DN_NB; ++j)
    if (j < nb) row[(int64_t)j * lda] = w[j];
}

// ---- generic column-major tile GEMM:  C (M x N) -= op(A) * op(B)   -------------------------------------------------
//   TA == 0: A is M x K (lda), element (i,k) = A[k*lda + i];   TA == 1: A is K x M, element (i,k) = A[i*lda + k]
//   TB == 0: B is K x N (ldb), element (k,j) = B[j*ldb + k];   TB == 1: B is N x K, element (k,j) = B[k*ldb + j]
//   lower != 0: only tiles with i-tile >= j-tile are computed (SYRK-style trailing update)
//   member blockIdx.z of a batch: A + z * astride, B + z * bstride, C + z * cstride
constexpr int GM_T = 64, GM_K = 16;
template <int TA, int TB>
__global__ void __launch_bounds__(256) gemm_sub_kernel(int64_t M, int64_t N, int K, const double* __restrict__ A,
                                                       int64_t lda, const double* __restrict__ B, int64_t ldb,
                                                       double* __restrict__ C, int64_t ldc, int lower,
                                                       const int* info, int64_t astride, int64_t bstride,
                                                       int64_t cstride) {
  if (info && *info != 0) return;
  if (lower && blockIdx.x < blockIdx.y) return;
  A += blockIdx.z * astride;
  B += blockIdx.z * bstride;
  C += blockIdx.z * cstride;
  __shared__ double sa[GM_K][GM_T + 4];
  __shared__ double sb[GM_K][GM_T + 4];
  const int64_t i0 = (int64_t)blockIdx.x * GM_T, j0 = (int64_t)blockIdx.y * GM_T;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;  // 16 x 16 threads, 4x4 outputs each
  double acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
  for (int k0 = 0; k0 < K; k0 += GM_K) {
    for (int t = threadIdx.x; t < GM_T * GM_K; t += 256) {
      int i, k;
      if (TA == 0) { i = t % GM_T; k = t / GM_T; } else { k = t % GM_K; i = t / GM_K; }
      const int64_t gi = i0 + i;
      const int gk = k0 + k;
      double v = 0.0;
      if (gi < M && gk < K) v = (TA == 0) ? A[(int64_t)gk * lda + gi] : A[gi * lda + gk];
      sa[k][i] = v;
    }
    for (int t = threadIdx.x; t < GM_T * GM_K; t += 256) {
      int j, k;
      if (TB == 1) { j = t % GM_T; k = t / GM_T; } else { k = t % GM_K; j = t / GM_K; }
      const int64_t gj = j0 + j;
      const int gk = k0 + k;
      double v = 0.0;
      if (gj < N && gk < K) v = (TB == 1) ? B[(int64_t)gk * ldb + gj] : B[gj * ldb + gk];
      sb[k][j] = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < GM_K; ++k) {
      double a[4], b[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) { a[e] = sa[k][tx + 16 * e]; b[e] = sb[k][ty + 16 * e]; }
#pragma unroll
      for (int e = 0; e < 4; ++e)
#pragma unroll
        for (int f = 0; f < 4; ++f) acc[e][f] += a[e] * b[f];
    }
    __syncthreads();
  }
#pragma unroll
  for (int f = 0; f < 4; ++f)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int64_t gi = i0 + tx + 16 * e, gj = j0 + ty + 16 * f;
      if (gi < M && gj < N && (!lower || gi >= gj)) C[gj * ldc + gi] -= acc[e][f];
    }
}

// ---- triangular solves with the diagonal block for a slab of right-hand sides --------------------------------------
// forward: X_k <- L_kk^-1 X_k ; backward: X_k <- L_kk^-T X_k.  One thread per RHS column; L_kk in shared memory.
// (member blockIdx.y of a batch: L + y * lstride, X + y * xstride)
__global__ void __launch_bounds__(128) trsv_block_kernel(const double* __restrict__ L, int64_t ldl, int nb,
                                                         double* __restrict__ X, int64_t ldx, int64_t nrhs,
                                                         int backward, int64_t lstride, int64_t xstride) {
  __shared__ double l[DN_NB][DN_NB + 1];
  L += blockIdx.y * lstride;
  X += blockIdx.y * xstride;
  for (int t = threadIdx.x; t < nb * nb; t += blockDim.x) {
    const int i = t % nb, j = t / nb;
    l[i][j] = L[(int64_t)j * ldl + i];
  }
  __syncthreads();
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nrhs) return;
  double* x = X + c * ldx;
  double w[DN_NB];
#pragma unroll
  for (int j = 0; j < DN_NB; ++j) w[j] = (j < nb) ? x[j] : 0.0;
  if (!backward) {
#pragma unroll
    for (int j = 0; j < DN_NB; ++j)
      if (j < nb) {
        double s = w[j];
#pragma unroll
        for (int q = 0; q < j; ++q) s -= l[j][q] * w[q];
        w[j] = s / l[j][j];
      }
  } else {
#pragma unroll
    for (int j = DN_NB - 1; j >= 0; --j)
      if (j < nb) {
        double s = w[j];
#pragma unroll
        for (int q = j + 1; q < DN_NB; ++q)
          if (q < nb) s -= l[q][j] * w[q];
        w[j] = s / l[j][j];
      }
  }
#pragma unroll
  for (int j = 0; j < DN_NB; ++j)
    if (j < nb) x[j] = w[j];
}

// ---- few right-hand sides (log_likelihood's single solve, predict's alpha): one launch per 64-column block ---------
// The generic path above spends ~30 us per block in a one-thread-per-RHS substitution; with 1..8 right-hand sides the
// solve is a chain of n/64 dependent steps whose useful work is reading L once (8 n^2 / 2 bytes per sweep), so every
// step is ONE launch: each CTA redundantly solves the 64 x 64 diagonal block with a warp per right-hand side (two
// entries per lane, pivots broadcast by shuffle) and then applies it to its own 256 rows (forward) or 256 columns
// (backward) of the panel.  The solved block goes to a second buffer so that no CTA reads entries another one is
// writing: forward reads B and writes Y, backward reads Y and writes the result back into B.
constexpr int DS_MAX_RHS = 8;
constexpr int DS_ROWS = 256;   // rows of the panel per CTA (forward)
constexpr int DS_COLS = 64;    // columns of the panel per CTA (backward)

// diagonal block (identity-padded to 64 x 64) and the reciprocals of its diagonal
__device__ __forceinline__ void load_diag_block(double (*l)[DN_NB + 1], double* rl, const double* __restrict__ Lkk,
                                                int64_t ld, int nb) {
  for (int t = threadIdx.x; t < DN_NB * DN_NB; t += blockDim.x) {
    const int i = t % DN_NB, j = t / DN_NB;
    l[i][j] = (i < nb && j < nb) ? Lkk[(int64_t)j * ld + i] : (i == j ? 1.0 : 0.0);
  }
  if (threadIdx.x < DN_NB) rl[threadIdx.x] = (threadIdx.x < nb) ? 1.0 / Lkk[(int64_t)threadIdx.x * ld + threadIdx.x] : 1.0;
}

// warp-level substitution with the 64 x 64 block in shared memory; entries (lane, lane + 32) of the vector per lane
__device__ __forceinline__ void warp_trsv_lower(const double (*l)[DN_NB + 1], const double* rl, int nb, int lane,
                                                double& w0, double& w1) {
  for (int j = 0; j < nb; ++j) {  // L x = b
    const double xj = __shfl_sync(0xffffffffu, (j < 32) ? w0 : w1, j & 31) * rl[j];
    if (j < 32) {
      if (lane == j) w0 = xj; else if (lane > j) w0 = fma(-l[lane][j], xj, w0);
      w1 = fma(-l[lane + 32][j], xj, w1);
    } else {
      const int jj = j - 32;
      if (lane == jj) w1 = xj; else if (lane > jj) w1 = fma(-l[lane + 32][j], xj, w1);
    }
  }
}
__device__ __forceinline__ void warp_trsv_lower_t(const double (*l)[DN_NB + 1], const double* rl, int nb, int lane,
                                                  double& w0, double& w1) {
  for (int j = nb - 1; j >= 0; --j) {  // L^T x = y
    const double xj = __shfl_sync(0xffffffffu, (j < 32) ? w0 : w1, j & 31) * rl[j];
    if (j >= 32) {
      const int jj = j - 32;
      if (lane == jj) w1 = xj; else if (lane < jj) w1 = fma(-l[j][lane + 32], xj, w1);
      w0 = fma(-l[j][lane], xj, w0);
    } else {
      if (lane == j) w0 = xj; else if (lane < j) w0 = fma(-l[j][lane], xj, w0);
    }
  }
}

// step k0 of  L y = b :  Y[k0:k0+nb] = L_kk^-1 B[k0:k0+nb] ;  B[k0+nb:] -= L[k0+nb:, k0:k0+nb] Y[k0:k0+nb]
// Member blockIdx.y of a batch solves with L + blockIdx.y * lstride on B, Y + blockIdx.y * vstride.
template <int NR>
__global__ void __launch_bounds__(DS_ROWS) trsv_fwd_step_kernel(const double* __restrict__ L, int64_t ld, int64_t n,
                                                                int64_t k0, int nb, double* __restrict__ B, int64_t ldb,
                                                                double* __restrict__ Y, int64_t ldy, int nrhs,
                                                                int64_t lstride, int64_t vstride) {
  __shared__ double l[DN_NB][DN_NB + 1];
  __shared__ double rl[DN_NB];
  __shared__ double xs[DS_MAX_RHS][DN_NB];
  L += blockIdx.y * lstride;
  B += blockIdx.y * vstride;
  Y += blockIdx.y * vstride;
  // this thread's row of the panel: the 64 loads are issued first so that they are in flight during the substitution
  const int64_t row = k0 + nb + (int64_t)blockIdx.x * DS_ROWS + threadIdx.x;
  double v[DN_NB];
  {
    const double* a = L + k0 * ld + (row < n ? row : k0);
#pragma unroll
    for (int q = 0; q < DN_NB; ++q) v[q] = (q < nb && row < n) ? a[(int64_t)q * ld] : 0.0;
  }
  load_diag_block(l, rl, L + k0 * ld + k0, ld, nb);
  for (int t = threadIdx.x; t < DS_MAX_RHS * DN_NB; t += blockDim.x) xs[t / DN_NB][t % DN_NB] = 0.0;
  __syncthreads();
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (w < nrhs) {
    const double* b = B + (int64_t)w * ldb + k0;
    double w0 = (lane < nb) ? b[lane] : 0.0, w1 = (lane + 32 < nb) ? b[lane + 32] : 0.0;
    warp_trsv_lower(l, rl, nb, lane, w0, w1);
    xs[w][lane] = w0; xs[w][lane + 32] = w1;
  }
  __syncthreads();
  if (blockIdx.x == 0)
    for (int t = threadIdx.x; t < nrhs * nb; t += blockDim.x) Y[(int64_t)(t / nb) * ldy + k0 + t % nb] = xs[t / nb][t % nb];
  if (row >= n) return;
  double acc[NR];
#pragma unroll
  for (int c = 0; c < NR; ++c) acc[c] = 0.0;
#pragma unroll
  for (int q = 0; q < DN_NB; ++q) {
#pragma unroll
    for (int c = 0; c < NR; ++c) acc[c] = fma(v[q], xs[c][q], acc[c]);
  }
#pragma unroll
  for (int c = 0; c < NR; ++c)
    if (c < nrhs) B[(int64_t)c * ldb + row] -= acc[c];
}

// step k0 of  L^T x = y :  X[k0:k0+nb] = L_kk^-T Y[k0:k0+nb] ;  Y[0:k0] -= L[k0:k0+nb, 0:k0]^T X[k0:k0+nb]
// The CTA's 64 columns of the panel (64 x 64, each column 512 contiguous bytes) are staged through shared memory with
// all loads in flight at once; then one thread per (column, right-hand side) takes the dot product.
// (member blockIdx.y of a batch: L + blockIdx.y * lstride, Y and X + blockIdx.y * vstride)
template <int NR>
__global__ void __launch_bounds__(256) trsv_bwd_step_kernel(const double* __restrict__ L, int64_t ld, int64_t k0,
                                                            int nb, double* __restrict__ Y, int64_t ldy,
                                                            double* __restrict__ X, int64_t ldx, int nrhs,
                                                            int64_t lstride, int64_t vstride) {
  L += blockIdx.y * lstride;
  Y += blockIdx.y * vstride;
  X += blockIdx.y * vstride;
  extern __shared__ __align__(16) double bwd_smem[];  // 71 KB: above the 48 KB static limit, opted in by the launcher
  double (*l)[DN_NB + 1] = reinterpret_cast<double (*)[DN_NB + 1]>(bwd_smem);
  double (*tile)[DN_NB + 1] = reinterpret_cast<double (*)[DN_NB + 1]>(bwd_smem + DN_NB * (DN_NB + 1));  // tile[c][q] = L[k0 + q, c_begin + c]
  double* rl = bwd_smem + (DN_NB + DS_COLS) * (DN_NB + 1);
  double (*xs)[DN_NB] = reinterpret_cast<double (*)[DN_NB]>(rl + DN_NB);
  const int64_t c_begin = (int64_t)blockIdx.x * DS_COLS;
  const int nc = (int)max((int64_t)0, min((int64_t)DS_COLS, k0 - c_begin));
  for (int t = threadIdx.x; t < DS_COLS * DN_NB; t += blockDim.x) {
    const int q = t % DN_NB, c = t / DN_NB;
    tile[c][q] = (c < nc && q < nb) ? L[(c_begin + c) * ld + k0 + q] : 0.0;
  }
  load_diag_block(l, rl, L + k0 * ld + k0, ld, nb);
  for (int t = threadIdx.x; t < DS_MAX_RHS * DN_NB; t += blockDim.x) xs[t / DN_NB][t % DN_NB] = 0.0;
  __syncthreads();
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (w < nrhs) {
    const double* y = Y + (int64_t)w * ldy + k0;
    double w0 = (lane < nb) ? y[lane] : 0.0, w1 = (lane + 32 < nb) ? y[lane + 32] : 0.0;
    warp_trsv_lower_t(l, rl, nb, lane, w0, w1);
    xs[w][lane] = w0; xs[w][lane + 32] = w1;
  }
  __syncthreads();
  if (blockIdx.x == 0)
    for (int t = threadIdx.x; t < nrhs * nb; t += blockDim.x) X[(int64_t)(t / nb) * ldx + k0 + t % nb] = xs[t / nb][t % nb];
  // thread (c, r0): column c of this CTA's slab, right-hand sides r0, r0 + 4, ...
  const int c = threadIdx.x % DS_COLS, r0 = threadIdx.x / DS_COLS;
  if (c >= nc) return;
#pragma unroll
  for (int rr = 0; rr < (NR + 3) / 4; ++rr) {
    const int r = r0 + 4 * rr;
    if (r < nrhs) {
      double s = 0.0;
#pragma unroll 16
      for (int q = 0; q < DN_NB; ++q) s = fma(tile[c][q], xs[r][q], s);
      Y[(int64_t)r * ldy + c_begin + c] -= s;
    }
  }
}

// one CTA per matrix: member blockIdx.x of a batch reads A + blockIdx.x * mstride and writes out[blockIdx.x]
__global__ void logdet_diag_kernel(const double* __restrict__ A, int64_t lda, int64_t n, double* out, int64_t mstride) {
  __shared__ double red[32];
  A += blockIdx.x * mstride;
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) s += log(A[i * lda + i]);
  s = block_sum(s, red);
  if (threadIdx.x == 0) out[blockIdx.x] = 2.0 * s;
}
__global__ void dot2_kernel(const double* __restrict__ a, const double* __restrict__ b, int64_t n, double* out) {
  __shared__ double red[32];
  double s = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    s += a[i] * b[i];
  s = block_sum(s, red);
  if (threadIdx.x == 0) atomicAdd(out, s);
}
// out[b] = r_b . x_b, one CTA per member, summed in a fixed order (no atomics): repeated calls give the same bits
__global__ void dot_rows_kernel(const double* __restrict__ r, const double* __restrict__ x, int64_t n,
                                double* __restrict__ out) {
  __shared__ double red[32];
  const double* a = r + blockIdx.x * n;
  const double* b = x + blockIdx.x * n;
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) s = fma(a[i], b[i], s);
  s = block_sum(s, red);
  if (threadIdx.x == 0) out[blockIdx.x] = s;
}
__global__ void square2_kernel(const double* __restrict__ yerr, double* __restrict__ diag, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    diag[i] = yerr[i] * yerr[i];
}
// b[i] = a[i] + b[i]: the batched draws' mean, K(x*, x) alpha plus the mean model at x*, one IEEE add per entry as
// GP.sample_conditional's host sum
__global__ void add_into_kernel(const double* __restrict__ a, double* __restrict__ b, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    b[i] = a[i] + b[i];
}
// A += 1/2 (beta alpha^T + alpha beta^T) over the whole n x n A (bgp_dense_loo_terms: A = -K^-1 diag(c) K^-1 before).
// Every rounding is explicit, so A stays exactly symmetric and A_ii = -M_ii + alpha_i beta_i.
// (member blockIdx.y of a batch: A + y * n^2, alpha and beta + y * n)
__global__ void loo_form_a_kernel(double* __restrict__ A, int64_t n, const double* __restrict__ alpha,
                                  const double* __restrict__ beta) {
  const int64_t total = n * n;
  A += blockIdx.y * total;
  alpha += blockIdx.y * n;
  beta += blockIdx.y * n;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t j = t / n, i = t - j * n;
    const double sym = __dadd_rn(__dmul_rn(beta[i], alpha[j]), __dmul_rn(alpha[i], beta[j]));
    A[t] = __dadd_rn(A[t], __dmul_rn(0.5, sym));
  }
}
// `members` matrices of order n back to back; a single call passes one member
static int loo_form_a_members(double* A, int64_t n, const double* alpha, const double* beta, int members,
                              cudaStream_t s) {
  loo_form_a_kernel<<<dim3((unsigned)std::min<int64_t>((n * n + 255) / 256, 16 * (int64_t)num_sms()), (unsigned)members),
                      256, 0, s>>>(A, n, alpha, beta);
  BGP_LAUNCH_CHECK();
  return BGP_OK;
}
// out (nr x n, row-major) = r (nr x n, row-major) @ U with U = L^T:  out[a][j] = sum_{i<=j} r[a][i] L[j][i]
__global__ void apply_sqrt_kernel(const double* __restrict__ L, int64_t n, const double* __restrict__ r, int64_t nr,
                                  double* __restrict__ out) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t a = blockIdx.y;
  if (j >= n) return;
  double s = 0.0;
  for (int64_t i = 0; i <= j; ++i) s += r[a * n + i] * L[i * n + j];  // L[j][i] column-major = L[i*n + j]
  out[a * n + j] = s;
}

}  // namespace bgp

using namespace bgp;

struct bgp_dense {
  cudaStream_t s = nullptr;
  cudaEvent_t ev[4] = {nullptr};
  int64_t n = 0;
  bool computed = false;
  double log_det = 0.0;
  DevBuf<DevProgram> d_prog;
  DevBuf<double> d_x, d_yerr, d_diag, d_A, d_rhs, d_scalar;
  DevBuf<double> d_tmp;              // second buffer of the few-RHS solve
  DevBuf<double> d_inv, d_gscratch;  // grad_terms: K^-1 (n x n) and the contraction partials
  DevBuf<unsigned> d_which;
  bool has_inputs = false;           // d_x / d_prog describe the factor in d_A (false after import_factor)
  int ndim = 0, n_params = 0;
  DevProgram prog;                   // host copy of d_prog (its shape selects the x-gradient evaluator)
  DevBuf<int> d_info;
  DevBuf<GemmDesc> d_gdesc;
  double t_ms[2] = {0, 0};
};

// outer block width (a multiple of DN_NB); BGP_DENSE_OB overrides the default for tuning runs and for tests that run
// every update level at small n.  Read at every compute(), like the other diagnostic switches.
static int64_t dense_outer_block() {
  int64_t ob = DN_OB;
  if (const char* e = getenv("BGP_DENSE_OB")) {
    const long v = atol(e);
    if (v >= DN_NB && v <= 4096 && v % DN_NB == 0) ob = v;
  }
  return ob;
}

// Blocked right-looking Cholesky with DELAYED trailing updates on three nested block sizes (64 | DN_MB | OB): after the
// panel ending at column e, the rank-64 update touches only the rest of the current DN_MB block; when e closes a DN_MB
// block its accumulated rank-DN_MB update touches the rest of the current OB block; when e closes an OB block the
// rank-OB update touches everything to the right.  Almost all flops therefore run as GEMMs with K = OB, whose
// read-modify-write epilogue of C is amortised over 16x more tensor work than at K = 64.
static int64_t dense_mid_block(int64_t OB) {
  int64_t mb = DN_MB;
  if (const char* e = getenv("BGP_DENSE_MB")) {
    const long v = atol(e);
    if (v >= DN_NB && v % DN_NB == 0) mb = v;
  }
  return (mb < OB && OB % mb == 0) ? mb : OB;
}

// `members` factorisations of the same order n run together: member m's matrix is A + m * mstride, its info word
// info[m]; every step is one launch for all of them (the GEMM descriptors of a step are consecutive, one per member,
// and go through grid.z).  gemm_info: the word the trailing updates test before running (a single factorisation
// passes its info word so that nothing runs after a failed pivot; a batch passes nullptr, so a failed member's updates
// run on its own slab's garbage, which no other member reads).
int bgp::dense_potrf_members(double* A, int64_t n, int64_t mstride, int members, int* info, const int* gemm_info,
                             DevBuf<GemmDesc>& gdesc, cudaStream_t s) {
  // all trailing-update descriptors of the factorisation, uploaded once
  std::vector<GemmDesc> descs;
  struct Step { int64_t k0; int nb; int64_t rem; int desc[3]; };
  std::vector<Step> steps;
  const int64_t OB = dense_outer_block();
  const int64_t MB = dense_mid_block(OB);
  // C[e:n, e:cend) -= L[e:n, b:e) L[e:cend, b:e)^T   (lower part only)
  auto add_update = [&](int64_t b, int64_t e, int64_t cend) -> int {
    if (e >= n || cend <= e || e <= b) return -1;
    const int first = (int)descs.size();
    for (int m = 0; m < members; ++m) {
      double* Am = A + m * mstride;
      GemmDesc d;
      const double* P = Am + b * n + e;         // rows e.., columns b..e of the factor
      d.A = P; d.lda = n; d.B = P; d.ldb = n;   // B' = P^T restricted to the first (cend - e) rows of P
      d.C = Am + e * n + e; d.ldc = n;
      d.M = (int)(n - e); d.N = (int)(cend - e); d.K = (int)(e - b); d.mode = GD_SUB | GD_LOWER;
      descs.push_back(d);
    }
    return first;
  };
  for (int64_t j0 = 0; j0 < n; j0 += DN_NB) {
    Step st;
    st.k0 = j0; st.nb = (int)std::min<int64_t>(DN_NB, n - j0); st.rem = n - j0 - st.nb;
    const int64_t e = j0 + st.nb;
    const int64_t mb0 = (j0 / MB) * MB, mb1 = std::min(n, mb0 + MB);  // the DN_MB block holding this panel
    const int64_t ob0 = (j0 / OB) * OB, ob1 = std::min(n, ob0 + OB);  // the OB block holding it
    st.desc[0] = add_update(j0, e, mb1);
    st.desc[1] = (e == mb1 && MB < OB) ? add_update(mb0, e, ob1) : -1;
    st.desc[2] = (e == ob1) ? add_update(ob0, e, n) : -1;
    steps.push_back(st);
  }
  BGP_TRY(gdesc.reserve(std::max<size_t>(descs.size(), 1), s));
  if (!descs.empty())
    BGP_CUDA(cudaMemcpyAsync(gdesc.p, descs.data(), sizeof(GemmDesc) * descs.size(), cudaMemcpyHostToDevice, s));
  for (const Step& st : steps) {
    double* Akk = A + st.k0 * n + st.k0;
    potf2_kernel<<<dim3(1, (unsigned)members), DN_NB, 0, s>>>(Akk, n, st.nb, info, (int)st.k0, mstride);
    BGP_LAUNCH_CHECK();
    if (st.rem <= 0) break;
    trsm_panel_kernel<<<dim3((unsigned)((st.rem + 127) / 128), (unsigned)members), 128, 0, s>>>(Akk, n, st.rem, st.nb,
                                                                                                info, mstride);
    BGP_LAUNCH_CHECK();
    for (int l = 0; l < 3; ++l)
      if (st.desc[l] >= 0)
        BGP_TRY((gemm_dmma_launch<false, false>(gdesc.p + st.desc[l], members, descs[st.desc[l]].M, descs[st.desc[l]].N, gemm_info, s)));
  }
  return BGP_OK;
}

static int dense_potrf(bgp_dense* h) {
  return dense_potrf_members(h->d_A.p, h->n, 0, 1, h->d_info.p, h->d_info.p, h->d_gdesc, h->s);
}

// X (n x nrhs, column-major ldx) <- K^-1 X on the device
constexpr size_t DS_BWD_SMEM = sizeof(double) * ((DN_NB + DS_COLS) * (DN_NB + 1) + DN_NB + DS_MAX_RHS * DN_NB);

// X <- K^-1 X for `members` factors of order n at once (member m: L + m * lstride, X and the scratch Y (n x nrhs,
// leading dimension n) + m * vstride); a single solve passes members = 1.
static int potrs_small_members(const double* L, int64_t n, double* X, int nrhs, int64_t ldx, double* Y, int members,
                               int64_t lstride, int64_t vstride, cudaStream_t s) {
  // (the attribute is per device / context: set it on every call, it is cheap)
  cudaFuncSetAttribute(trsv_bwd_step_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DS_BWD_SMEM);
    cudaFuncSetAttribute(trsv_bwd_step_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DS_BWD_SMEM);
    cudaFuncSetAttribute(trsv_bwd_step_kernel<DS_MAX_RHS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DS_BWD_SMEM);
  const unsigned mb = (unsigned)members;
  for (int64_t k0 = 0; k0 < n; k0 += DN_NB) {
    const int nb = (int)std::min<int64_t>(DN_NB, n - k0);
    const int64_t rem = n - k0 - nb;
    const dim3 g((unsigned)std::max<int64_t>(1, (rem + DS_ROWS - 1) / DS_ROWS), mb);
    if (nrhs == 1) trsv_fwd_step_kernel<1><<<g, DS_ROWS, 0, s>>>(L, n, n, k0, nb, X, ldx, Y, n, nrhs, lstride, vstride);
    else if (nrhs <= 4) trsv_fwd_step_kernel<4><<<g, DS_ROWS, 0, s>>>(L, n, n, k0, nb, X, ldx, Y, n, nrhs, lstride, vstride);
    else trsv_fwd_step_kernel<DS_MAX_RHS><<<g, DS_ROWS, 0, s>>>(L, n, n, k0, nb, X, ldx, Y, n, nrhs, lstride, vstride);
    BGP_LAUNCH_CHECK();
  }
  for (int64_t k0 = ((n - 1) / DN_NB) * DN_NB; k0 >= 0; k0 -= DN_NB) {
    const int nb = (int)std::min<int64_t>(DN_NB, n - k0);
    const dim3 g((unsigned)std::max<int64_t>(1, (k0 + DS_COLS - 1) / DS_COLS), mb);
    if (nrhs == 1) trsv_bwd_step_kernel<1><<<g, 256, DS_BWD_SMEM, s>>>(L, n, k0, nb, Y, n, X, ldx, nrhs, lstride, vstride);
    else if (nrhs <= 4) trsv_bwd_step_kernel<4><<<g, 256, DS_BWD_SMEM, s>>>(L, n, k0, nb, Y, n, X, ldx, nrhs, lstride, vstride);
    else trsv_bwd_step_kernel<DS_MAX_RHS><<<g, 256, DS_BWD_SMEM, s>>>(L, n, k0, nb, Y, n, X, ldx, nrhs, lstride, vstride);
    BGP_LAUNCH_CHECK();
  }
  return BGP_OK;
}

// X (n x nrhs, column-major ldx) <- L^-1 X: the forward half of dense_potrs_dev (predictive variance / covariance need
// only W = L^-1 K(x, x*), since K(x*, x) K^-1 K(x, x*) = W^T W).  `members` factors at once: member m solves with
// L + m * lstride on X + m * xstride; a single solve passes one member and zero strides.  Few right-hand sides go
// through the one-launch step kernels, which leave the result in Y; Y has X's layout (leading dimension ldy, member
// stride xstride, so ldy >= (members - 1) * xstride + n) and is copied back into X.
static int trsm_fwd_members(const double* L, int64_t n, int64_t lstride, double* X, int64_t nrhs, int64_t ldx,
                            int64_t xstride, int members, double* Y, int64_t ldy, cudaStream_t s) {
  const unsigned mb = (unsigned)members;
  if (nrhs <= DS_MAX_RHS) {
    for (int64_t k0 = 0; k0 < n; k0 += DN_NB) {
      const int nb = (int)std::min<int64_t>(DN_NB, n - k0);
      const int64_t rem = n - k0 - nb;
      const dim3 g((unsigned)std::max<int64_t>(1, (rem + DS_ROWS - 1) / DS_ROWS), mb);
      const int nr = (int)nrhs;
      if (nr == 1) trsv_fwd_step_kernel<1><<<g, DS_ROWS, 0, s>>>(L, n, n, k0, nb, X, ldx, Y, ldy, nr, lstride, xstride);
      else if (nr <= 4) trsv_fwd_step_kernel<4><<<g, DS_ROWS, 0, s>>>(L, n, n, k0, nb, X, ldx, Y, ldy, nr, lstride, xstride);
      else trsv_fwd_step_kernel<DS_MAX_RHS><<<g, DS_ROWS, 0, s>>>(L, n, n, k0, nb, X, ldx, Y, ldy, nr, lstride, xstride);
      BGP_LAUNCH_CHECK();
    }
    BGP_CUDA(cudaMemcpy2DAsync(X, sizeof(double) * ldx, Y, sizeof(double) * ldy,
                               sizeof(double) * ((int64_t)(members - 1) * xstride + n), nrhs, cudaMemcpyDeviceToDevice, s));
    return BGP_OK;
  }
  const unsigned cb = (unsigned)((nrhs + 127) / 128);
  for (int64_t k0 = 0; k0 < n; k0 += DN_NB) {
    const int nb = (int)std::min<int64_t>(DN_NB, n - k0);
    trsv_block_kernel<<<dim3(cb, mb), 128, 0, s>>>(L + k0 * n + k0, n, nb, X + k0, ldx, nrhs, 0, lstride, xstride);
    BGP_LAUNCH_CHECK();
    const int64_t rem = n - k0 - nb;
    if (rem <= 0) break;
    dim3 grid((unsigned)((rem + GM_T - 1) / GM_T), (unsigned)((nrhs + GM_T - 1) / GM_T), mb);
    gemm_sub_kernel<0, 0><<<grid, 256, 0, s>>>(rem, nrhs, nb, L + k0 * n + k0 + nb, n, X + k0, ldx, X + k0 + nb, ldx, 0,
                                               nullptr, lstride, xstride, xstride);
    BGP_LAUNCH_CHECK();
  }
  return BGP_OK;
}

// X <- K^-1 X for `members` factors of order n (member m: L + m * lstride, X + m * xstride); a single solve passes one
// member and zero strides.  Up to DS_MAX_RHS right-hand sides go through the one-launch step kernels with the scratch Y
// (members blocks of xstride >= n * nrhs doubles); more through the forward sweep of trsm_fwd_members and the
// backward sweep below.
// X (n x nrhs, column-major ldx) <- L^-T X in place, block by block from the bottom: the backward half of
// potrs_members for more than DS_MAX_RHS right-hand sides (any nrhs works).  Member m: L + m * lstride, X + m * xstride.
static int trsm_bwd_block_members(const double* L, int64_t n, int64_t lstride, double* X, int64_t nrhs, int64_t ldx,
                                  int64_t xstride, int members, cudaStream_t s) {
  const unsigned mb = (unsigned)members;
  const unsigned cb = (unsigned)((nrhs + 127) / 128);
  const int64_t last = ((n - 1) / DN_NB) * DN_NB;
  for (int64_t k0 = last; k0 >= 0; k0 -= DN_NB) {  // backward: L^T x = y
    const int nb = (int)std::min<int64_t>(DN_NB, n - k0);
    trsv_block_kernel<<<dim3(cb, mb), 128, 0, s>>>(L + k0 * n + k0, n, nb, X + k0, ldx, nrhs, 1, lstride, xstride);
    BGP_LAUNCH_CHECK();
    if (k0 == 0) break;
    // X[0:k0] -= L[k0:k0+nb, 0:k0]^T X[k0:k0+nb]
    dim3 grid((unsigned)((k0 + GM_T - 1) / GM_T), (unsigned)((nrhs + GM_T - 1) / GM_T), mb);
    gemm_sub_kernel<1, 0><<<grid, 256, 0, s>>>(k0, nrhs, nb, L + k0, n, X + k0, ldx, X, ldx, 0, nullptr, lstride, xstride,
                                               xstride);
    BGP_LAUNCH_CHECK();
  }
  return BGP_OK;
}

static int potrs_members(const double* L, int64_t n, int64_t lstride, double* X, int64_t nrhs, int64_t ldx,
                         int64_t xstride, int members, double* Y, cudaStream_t s) {
  if (nrhs <= DS_MAX_RHS) return potrs_small_members(L, n, X, (int)nrhs, ldx, Y, members, lstride, xstride, s);
  BGP_TRY(trsm_fwd_members(L, n, lstride, X, nrhs, ldx, xstride, members, nullptr, 0, s));  // forward: L y = b
  return trsm_bwd_block_members(L, n, lstride, X, nrhs, ldx, xstride, members, s);
}

static int dense_potrs_dev(bgp_dense* h, double* X, int64_t nrhs, int64_t ldx) {
  if (nrhs <= DS_MAX_RHS) BGP_TRY(h->d_tmp.reserve((size_t)h->n * DS_MAX_RHS, h->s));
  return potrs_members(h->d_A.p, h->n, 0, X, nrhs, ldx, 0, 1, h->d_tmp.p, h->s);
}

static int dense_trsm_fwd_dev(bgp_dense* h, double* X, int64_t nrhs, int64_t ldx) {
  if (nrhs <= DS_MAX_RHS) BGP_TRY(h->d_tmp.reserve((size_t)h->n * DS_MAX_RHS, h->s));
  return trsm_fwd_members(h->d_A.p, h->n, 0, X, nrhs, ldx, 0, 1, h->d_tmp.p, h->n, h->s);
}

// X (n x nrhs, column-major ldx) <- L^-T X: the backward half of potrs_members, so that trsm_fwd_members followed by
// this is K^-1.  `members` factors at once (member m: L + m * lstride, X + m * xstride); a single solve passes one member
// and zero strides.  Few right-hand sides go through the one-launch step kernels of potrs_small_members, which read the
// forward result from a copy in Y (X's layout: leading dimension ldy, member stride xstride, so ldy >= (members - 1) *
// xstride + n); more through trsm_bwd_block_members.
static int trsm_bwd_members(const double* L, int64_t n, int64_t lstride, double* X, int64_t nrhs, int64_t ldx,
                            int64_t xstride, int members, double* Y, int64_t ldy, cudaStream_t s) {
  if (nrhs > DS_MAX_RHS) return trsm_bwd_block_members(L, n, lstride, X, nrhs, ldx, xstride, members, s);
  const unsigned mb = (unsigned)members;
  BGP_CUDA(cudaMemcpy2DAsync(Y, sizeof(double) * ldy, X, sizeof(double) * ldx,
                             sizeof(double) * ((int64_t)(members - 1) * xstride + n), nrhs, cudaMemcpyDeviceToDevice, s));
  cudaFuncSetAttribute(trsv_bwd_step_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DS_BWD_SMEM);
  cudaFuncSetAttribute(trsv_bwd_step_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DS_BWD_SMEM);
  cudaFuncSetAttribute(trsv_bwd_step_kernel<DS_MAX_RHS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DS_BWD_SMEM);
  const int nr = (int)nrhs;
  for (int64_t k0 = ((n - 1) / DN_NB) * DN_NB; k0 >= 0; k0 -= DN_NB) {
    const int nb = (int)std::min<int64_t>(DN_NB, n - k0);
    const dim3 g((unsigned)std::max<int64_t>(1, (k0 + DS_COLS - 1) / DS_COLS), mb);
    if (nr == 1) trsv_bwd_step_kernel<1><<<g, 256, DS_BWD_SMEM, s>>>(L, n, k0, nb, Y, ldy, X, ldx, nr, lstride, xstride);
    else if (nr <= 4) trsv_bwd_step_kernel<4><<<g, 256, DS_BWD_SMEM, s>>>(L, n, k0, nb, Y, ldy, X, ldx, nr, lstride, xstride);
    else trsv_bwd_step_kernel<DS_MAX_RHS><<<g, 256, DS_BWD_SMEM, s>>>(L, n, k0, nb, Y, ldy, X, ldx, nr, lstride, xstride);
    BGP_LAUNCH_CHECK();
  }
  return BGP_OK;
}

// X (n x nrhs, column-major ldx) <- L^-T X on the handle's factor, the scratch Y in d_tmp
static int dense_trsm_bwd_dev(bgp_dense* h, double* X, int64_t nrhs, int64_t ldx) {
  if (nrhs <= DS_MAX_RHS) BGP_TRY(h->d_tmp.reserve((size_t)h->n * DS_MAX_RHS, h->s));
  return trsm_bwd_members(h->d_A.p, h->n, 0, X, nrhs, ldx, 0, 1, h->d_tmp.p, h->n, h->s);
}

// GP.predict's covariance at the ns test points xs (host) into dC (ns x ns on the device, allocated here): every W chunk
// stays resident (n*ns), then C = K** - W^T W (lower, mirrored: exactly symmetric).  P is the validated program of the
// prediction's kernel.  bgp_dense_predict copies dC out; bgp_dense_sample draws from it on the device.
static int dense_predict_cov_dev(bgp_dense* h, const DevProgram& P, const double* xs, int64_t ns, DevBuf<double>& dC) {
  const int64_t n = h->n;
  const int nd = h->ndim;
  cudaStream_t s = h->s;
  DevBuf<DevProgram> dprog;
  DevBuf<double> dxs, dW, scratch;
  DevBuf<GemmDesc> ddesc;
  BGP_TRY(upload_program(P, dprog, s));
  const int64_t c = std::min(ns, predict_chunk_cols(n, 1));
  BGP_TRY(dxs.alloc((size_t)ns * nd, s));
  BGP_TRY(dW.alloc((size_t)n * ns, s));
  BGP_TRY(dC.alloc((size_t)ns * ns, s));
  BGP_CUDA(cudaMemcpyAsync(dxs.p, xs, sizeof(double) * ns * nd, cudaMemcpyHostToDevice, s));
  BGP_TRY(kmat_symmetric_launch_auto(P, dprog.p, dxs.p, ns, nullptr, dC.p, ns, s));
  for (int64_t j0 = 0; j0 < ns; j0 += c) {
    const int64_t nc = std::min(c, ns - j0);
    BGP_TRY(kmat_general_launch_auto(P, dprog.p, dxs.p + j0 * nd, nc, h->d_x.p, n, dW.p + j0 * n, n, s));
    BGP_TRY(dense_trsm_fwd_dev(h, dW.p + j0 * n, nc, n));
  }
  return predict_gemm_sub(dW.p, n, dW.p, n, ns, ns, n, true, dC.p, ns, scratch, ddesc, s);
}

extern "C" {

int bgp_dense_create(bgp_dense_t** out) {
  *out = new (std::nothrow) bgp_dense();
  if (!*out) { set_error("out of host memory"); return BGP_ERR_NOMEM; }
  return BGP_OK;
}

void bgp_dense_destroy(bgp_dense_t* h) {
  if (!h) return;
  if (h->s) cudaStreamSynchronize(h->s);
  h->d_prog.release(); h->d_x.release(); h->d_yerr.release(); h->d_diag.release(); h->d_A.release();
  h->d_rhs.release(); h->d_scalar.release(); h->d_info.release(); h->d_gdesc.release();
  h->d_tmp.release(); h->d_inv.release(); h->d_gscratch.release(); h->d_which.release();
  if (h->s) {
    cudaStreamSynchronize(h->s);
    for (int i = 0; i < 4; ++i) cudaEventDestroy(h->ev[i]);
    cudaStreamDestroy(h->s);
  }
  delete h;
}

int bgp_dense_compute(bgp_dense_t* h, const bgp_kernel_spec_t* spec, const double* x, int64_t n, int32_t ndim,
                      const double* yerr) {
  if (!h) { set_error("null handle"); return BGP_ERR_INVALID; }
  h->computed = false;
  BGP_TRY(require_device());
  if (!h->s) {
    BGP_CUDA(cudaStreamCreateWithFlags(&h->s, cudaStreamNonBlocking));
    for (int i = 0; i < 4; ++i) BGP_CUDA(cudaEventCreate(&h->ev[i]));
  }
  DevProgram P;
  BGP_TRY(build_dev_program(spec, &P));
  if (P.ndim != ndim) { set_error("dimension mismatch: kernel ndim %d, input ndim %d", P.ndim, ndim); return BGP_ERR_DIM; }
  if (n <= 0) { set_error("invalid number of points"); return BGP_ERR_INVALID; }
  cudaStream_t s = h->s;
  h->n = n;
  h->has_inputs = false;
  h->ndim = ndim;
  h->n_params = P.n_params_total;
  h->prog = P;
  BGP_TRY(upload_program(P, h->d_prog, s));
  BGP_TRY(h->d_x.reserve((size_t)n * ndim, s));
  BGP_TRY(h->d_yerr.reserve((size_t)n, s));
  BGP_TRY(h->d_diag.reserve((size_t)n, s));
  BGP_TRY(h->d_A.reserve((size_t)n * n, s));
  BGP_TRY(h->d_info.reserve(1, s));
  BGP_TRY(h->d_scalar.reserve(2, s));
  BGP_CUDA(cudaMemcpyAsync(h->d_x.p, x, sizeof(double) * n * ndim, cudaMemcpyHostToDevice, s));
  BGP_CUDA(cudaMemcpyAsync(h->d_yerr.p, yerr, sizeof(double) * n, cudaMemcpyHostToDevice, s));
  BGP_CUDA(cudaMemsetAsync(h->d_info.p, 0, sizeof(int), s));
  square2_kernel<<<(unsigned)std::min<int64_t>((n + 255) / 256, 1184), 256, 0, s>>>(h->d_yerr.p, h->d_diag.p, n);
  BGP_LAUNCH_CHECK();
  BGP_CUDA(cudaEventRecord(h->ev[0], s));
  BGP_TRY(kmat_symmetric_launch_auto(P, h->d_prog.p, h->d_x.p, n, h->d_diag.p, h->d_A.p, n, s));
  BGP_CUDA(cudaEventRecord(h->ev[1], s));
  BGP_TRY(dense_potrf(h));
  logdet_diag_kernel<<<1, 1024, 0, s>>>(h->d_A.p, n, n, h->d_scalar.p, 0);
  BGP_LAUNCH_CHECK();
  BGP_CUDA(cudaEventRecord(h->ev[2], s));
  int info = 0;
  double ld = 0.0;
  BGP_CUDA(cudaMemcpyAsync(&info, h->d_info.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaMemcpyAsync(&ld, h->d_scalar.p, sizeof(double), cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  float ms = 0;
  cudaEventElapsedTime(&ms, h->ev[0], h->ev[1]); h->t_ms[0] = ms;
  cudaEventElapsedTime(&ms, h->ev[1], h->ev[2]); h->t_ms[1] = ms;
  if (info != 0) {
    set_error("%d-th leading minor of the array is not positive definite", info);
    return BGP_ERR_LINALG;
  }
  h->log_det = ld;
  h->computed = true;
  h->has_inputs = true;
  return BGP_OK;
}

int bgp_dense_computed(const bgp_dense_t* h) { return h && h->computed ? 1 : 0; }

int bgp_dense_log_determinant(const bgp_dense_t* h, double* out) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  *out = h->log_det;
  return BGP_OK;
}

int bgp_dense_apply_inverse(bgp_dense_t* h, double* b, int64_t nrhs, int64_t ldb) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  if (nrhs <= 0) return BGP_OK;
  if (ldb < h->n) { set_error("dimension mismatch: ldb < n"); return BGP_ERR_DIM; }
  const int64_t n = h->n;
  cudaStream_t s = h->s;
  const int64_t slab = std::max<int64_t>(1, std::min<int64_t>(nrhs, (int64_t)(1ull << 28) / n));
  BGP_TRY(h->d_rhs.reserve((size_t)n * slab, s));
  for (int64_t c0 = 0; c0 < nrhs; c0 += slab) {
    const int64_t nc = std::min(slab, nrhs - c0);
    BGP_CUDA(cudaMemcpy2DAsync(h->d_rhs.p, sizeof(double) * n, b + c0 * ldb, sizeof(double) * ldb, sizeof(double) * n, nc, cudaMemcpyHostToDevice, s));
    BGP_TRY(dense_potrs_dev(h, h->d_rhs.p, nc, n));
    BGP_CUDA(cudaMemcpy2DAsync(b + c0 * ldb, sizeof(double) * ldb, h->d_rhs.p, sizeof(double) * n, sizeof(double) * n, nc, cudaMemcpyDeviceToHost, s));
    BGP_CUDA(cudaStreamSynchronize(s));
  }
  return BGP_OK;
}

int bgp_dense_dot_solve(bgp_dense_t* h, const double* y, double* out) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  const int64_t n = h->n;
  cudaStream_t s = h->s;
  BGP_TRY(h->d_rhs.reserve((size_t)n * 2, s));
  double* yd = h->d_rhs.p;
  double* xd = h->d_rhs.p + n;
  BGP_CUDA(cudaMemcpyAsync(yd, y, sizeof(double) * n, cudaMemcpyHostToDevice, s));
  BGP_CUDA(cudaMemcpyAsync(xd, yd, sizeof(double) * n, cudaMemcpyDeviceToDevice, s));
  BGP_TRY(dense_potrs_dev(h, xd, 1, n));
  BGP_CUDA(cudaMemsetAsync(h->d_scalar.p + 1, 0, sizeof(double), s));
  dot2_kernel<<<(unsigned)std::min<int64_t>((n + 255) / 256, 592), 256, 0, s>>>(yd, xd, n, h->d_scalar.p + 1);
  BGP_LAUNCH_CHECK();
  BGP_CUDA(cudaMemcpyAsync(out, h->d_scalar.p + 1, sizeof(double), cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  return BGP_OK;
}

int bgp_dense_apply_sqrt(bgp_dense_t* h, const double* r, int64_t nr, double* out) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  const int64_t n = h->n;
  cudaStream_t s = h->s;
  if (nr <= 0) return BGP_OK;
  DevBuf<double> dr, dout;
  BGP_TRY(dr.alloc((size_t)nr * n, s));
  BGP_TRY(dout.alloc((size_t)nr * n, s));
  BGP_CUDA(cudaMemcpyAsync(dr.p, r, sizeof(double) * nr * n, cudaMemcpyHostToDevice, s));
  dim3 grid((unsigned)((n + 127) / 128), (unsigned)nr);
  apply_sqrt_kernel<<<grid, 128, 0, s>>>(h->d_A.p, n, dr.p, nr, dout.p);
  BGP_LAUNCH_CHECK();
  BGP_CUDA(cudaMemcpyAsync(out, dout.p, sizeof(double) * nr * n, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  return BGP_OK;
}

int bgp_dense_get_inverse(bgp_dense_t* h, double* out) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  const int64_t n = h->n;
  for (int64_t j = 0; j < n; ++j) {
    double* c = out + j * n;
    memset(c, 0, sizeof(double) * n);
    c[j] = 1.0;
  }
  return bgp_dense_apply_inverse(h, out, n, n);
}

// GP.fisher_information's rows (bgp_dense_fisher_terms): nv white-noise vectors (host, nv x n) and the outputs
struct FisherArgs {
  const double* v;
  int nv;
  double* rows_out;     // nrow x np
  double* rdiag_out;    // nrow x n
  double* prod_ms_out;  // nrow (may be NULL): device time of each row's products
};

// The Fisher rows from the resident K^-1 (see bgp_dense_fisher_terms).  Row by row, one n x n plane / product buffer P and
// one n x n T: a kernel row p builds dK_p into P, T = -K^-T dK_p and P = K^-T dK_p K^-1 (two GD_SUB products into zeroed
// targets, the second one lower-triangular and mirrored, with T consumed as stored); a white-noise row scales the rows of
// a copy of K^-1 in T by v and forms P = -K^-T diag(v) K^-1 (one lower product).  The contraction of bgp_dense_grad_terms
// then gives the row's kernel entries (cm = +1 or -1 for the sign of P) and diag(P), each row in its own fixed order.
static int dense_fisher_rows(bgp_dense* h, const uint32_t* which, int np, const FisherArgs& f) {
  const int64_t n = h->n;
  const int nd = h->ndim;
  cudaStream_t s = h->s;
  std::vector<int> krow;
  for (int q = 0; q < np; ++q)
    if (which[q]) krow.push_back(q);
  const int nk = (int)krow.size(), nrow = nk + f.nv;
  if (nrow == 0) return BGP_OK;
  DevBuf<double> dP, dT, dv, drows, drd, slices;
  DevBuf<GemmDesc> descs;
  BGP_TRY(dP.alloc((size_t)n * n, s));
  BGP_TRY(dT.alloc((size_t)n * n, s));
  if (f.nv) {
    BGP_TRY(dv.alloc((size_t)f.nv * n, s));
    BGP_CUDA(cudaMemcpyAsync(dv.p, f.v, sizeof(double) * f.nv * n, cudaMemcpyHostToDevice, s));
  }
  BGP_TRY(drows.alloc((size_t)std::max(nrow * np, 1), s));
  BGP_TRY(drd.alloc((size_t)nrow * n, s));
  const size_t bytes = sizeof(double) * (size_t)n * (size_t)n;
  for (int row = 0; row < nrow; ++row) {
    if (f.prod_ms_out) BGP_CUDA(cudaEventRecord(h->ev[0], s));
    double cm = 1.0;
    if (row < nk) {
      BGP_TRY(kmat_gradient_plane_launch(h->d_prog.p, np, krow[row], h->d_x.p, n, dP.p, n, s));
      BGP_CUDA(cudaMemsetAsync(dT.p, 0, bytes, s));
      BGP_TRY(predict_gemm_sub(h->d_inv.p, n, dP.p, n, n, n, n, false, dT.p, n, slices, descs, s));
      BGP_CUDA(cudaMemsetAsync(dP.p, 0, bytes, s));
      BGP_TRY(predict_gemm_sub_bt(h->d_inv.p, n, dT.p, n, n, n, n, true, dP.p, n, slices, descs, s));
    } else {
      BGP_CUDA(cudaMemcpyAsync(dT.p, h->d_inv.p, bytes, cudaMemcpyDeviceToDevice, s));
      BGP_TRY(scale_rows_launch(dT.p, n, n, n, dv.p + (int64_t)(row - nk) * n, false, s));
      BGP_CUDA(cudaMemsetAsync(dP.p, 0, bytes, s));
      BGP_TRY(predict_gemm_sub(h->d_inv.p, n, dT.p, n, n, n, n, true, dP.p, n, slices, descs, s));
      cm = -1.0;
    }
    if (f.prod_ms_out) {
      BGP_CUDA(cudaEventRecord(h->ev[1], s));
      BGP_CUDA(cudaEventSynchronize(h->ev[1]));
      float ms = 0.0f;
      BGP_CUDA(cudaEventElapsedTime(&ms, h->ev[0], h->ev[1]));
      f.prod_ms_out[row] = ms;
    }
    BGP_TRY(kmat_grad_contract_launch(h->d_prog.p, nd, np, h->d_which.p, h->d_x.p, n, dP.p, n, nullptr, 0.0, cm,
                                      drows.p + (int64_t)row * np, drd.p + (int64_t)row * n, h->d_gscratch, s));
  }
  if (np) BGP_CUDA(cudaMemcpyAsync(f.rows_out, drows.p, sizeof(double) * nrow * np, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaMemcpyAsync(f.rdiag_out, drd.p, sizeof(double) * nrow * n, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  return BGP_OK;
}

// With xgrad (bgp_dense_grad_x_terms) the call also forms dx (n x ndim, row-major) from the resident K^-1 after the
// contraction: grad_x_resident_launch turns it into alpha alpha^T - K^-1 and runs the x-gradient matvec over it.  A NULL
// `which` then skips the parameter contraction.  With fisher (bgp_dense_fisher_terms) it forms the Fisher rows from the
// resident K^-1 after the contraction; a NULL `r` then skips alpha and the contraction.
static int dense_grad_terms_impl(bgp_dense* h, const uint32_t* which, const double* r, double* alpha_out, double* g_out,
                                 double* diag_out, bool xgrad, double* dx_out, const FisherArgs* fisher = nullptr) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  if (!h->has_inputs) { set_error("the factor was imported: the handle holds no kernel/coordinates"); return BGP_ERR_NOT_COMPUTED; }
  const int64_t n = h->n;
  const int np = (xgrad && !which) ? 0 : h->n_params;
  if (np > 64) { set_error("gradient supports at most 64 hyper-parameters"); return BGP_ERR_INVALID; }
  const int nd = h->ndim;
  if (xgrad && nd > BGP_MAX_DIM) { set_error("input-coordinate gradients support at most %d dimensions (got %d)", BGP_MAX_DIM, nd); return BGP_ERR_INVALID; }
  if (fisher) {
    if (np && !which) { set_error("fisher_terms: which is required for a kernel with parameters"); return BGP_ERR_INVALID; }
    if (fisher->nv < 0 || (fisher->nv && !fisher->v)) { set_error("fisher_terms: invalid white-noise vectors"); return BGP_ERR_INVALID; }
    if (!fisher->rows_out || !fisher->rdiag_out) { set_error("fisher_terms: NULL output"); return BGP_ERR_INVALID; }
  } else if (!r) {
    set_error("r is NULL"); return BGP_ERR_INVALID;
  }
  cudaStream_t s = h->s;
  BGP_TRY(h->d_rhs.reserve((size_t)n * 2 + 64, s));
  double* alpha = h->d_rhs.p;
  double* dg = h->d_rhs.p + n;       // np <= 64 entries
  double* ddiag = h->d_rhs.p + n + 64;
  if (r) {
    BGP_CUDA(cudaMemcpyAsync(alpha, r, sizeof(double) * n, cudaMemcpyHostToDevice, s));
    BGP_TRY(dense_potrs_dev(h, alpha, 1, n));
    if (alpha_out) BGP_CUDA(cudaMemcpyAsync(alpha_out, alpha, sizeof(double) * n, cudaMemcpyDeviceToHost, s));
  }
  BGP_TRY(h->d_inv.reserve((size_t)n * n, s));
  BGP_TRY(fill_identity_launch(h->d_inv.p, n, s));
  BGP_TRY(dense_potrs_dev(h, h->d_inv.p, n, n));
  BGP_TRY(h->d_which.reserve(std::max(np, 1), s));
  if (np) BGP_CUDA(cudaMemcpyAsync(h->d_which.p, which, sizeof(unsigned) * np, cudaMemcpyHostToDevice, s));
  // kernel term of gp.py:457-466 and diag(alpha alpha^T - K^-1) for the white-noise term of gp.py:452-456
  if (r)
    BGP_TRY(kmat_grad_contract_launch(h->d_prog.p, h->ndim, np, h->d_which.p, h->d_x.p, n, h->d_inv.p, n, alpha, 1.0, -1.0,
                                      dg, diag_out ? ddiag : nullptr, h->d_gscratch, s));
  if (fisher) {
    if (r) {  // bgp_dense_grad_terms' outputs, queued before the rows
      if (np && g_out) BGP_CUDA(cudaMemcpyAsync(g_out, dg, sizeof(double) * np, cudaMemcpyDeviceToHost, s));
      if (diag_out) BGP_CUDA(cudaMemcpyAsync(diag_out, ddiag, sizeof(double) * n, cudaMemcpyDeviceToHost, s));
    }
    return dense_fisher_rows(h, which, np, *fisher);
  }
  DevBuf<double> ddx;
  if (xgrad) {
    BGP_TRY(ddx.alloc((size_t)n * nd, s));
    BGP_TRY(grad_x_resident_launch(h->prog, h->d_prog.p, h->d_x.p, n, h->d_inv.p, alpha, ddx.p, h->d_gscratch, s));
  }
  if (np && g_out) BGP_CUDA(cudaMemcpyAsync(g_out, dg, sizeof(double) * np, cudaMemcpyDeviceToHost, s));
  if (diag_out) BGP_CUDA(cudaMemcpyAsync(diag_out, ddiag, sizeof(double) * n, cudaMemcpyDeviceToHost, s));
  if (xgrad && dx_out) BGP_CUDA(cudaMemcpyAsync(dx_out, ddx.p, sizeof(double) * n * nd, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  return BGP_OK;
}

int bgp_dense_grad_terms(bgp_dense_t* h, const uint32_t* which, const double* r, double* alpha_out, double* g_out,
                         double* diag_out) {
  return dense_grad_terms_impl(h, which, r, alpha_out, g_out, diag_out, false, nullptr);
}

int bgp_dense_grad_x_terms(bgp_dense_t* h, const uint32_t* which, const double* r, double* alpha_out, double* g_out,
                           double* diag_out, double* dx_out) {
  return dense_grad_terms_impl(h, which, r, alpha_out, g_out, diag_out, true, dx_out);
}

int bgp_dense_fisher_terms(bgp_dense_t* h, const uint32_t* which, const double* r, const double* v, int32_t nv,
                           double* alpha_out, double* g_out, double* diag_out, double* rows_out, double* rdiag_out,
                           double* prod_ms_out) {
  const FisherArgs f{v, nv, rows_out, rdiag_out, prod_ms_out};
  return dense_grad_terms_impl(h, which, r, alpha_out, g_out, diag_out, false, nullptr, &f);
}

int bgp_dense_loo_terms(bgp_dense_t* h, const uint32_t* which, const double* r, double* alpha_out, double* d_out,
                        double* beta_out, double* g_out, double* diag_out) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  if (!h->has_inputs) { set_error("the factor was imported: the handle holds no kernel/coordinates"); return BGP_ERR_NOT_COMPUTED; }
  const int64_t n = h->n;
  const int np = h->n_params;
  const bool grad = beta_out || g_out || diag_out;
  if (grad && np > 64) { set_error("gradient supports at most 64 hyper-parameters"); return BGP_ERR_INVALID; }
  cudaStream_t s = h->s;
  BGP_TRY(h->d_rhs.reserve((size_t)n * 5 + 64, s));
  double* alpha = h->d_rhs.p;
  double* dg = h->d_rhs.p + n;  // np <= 64 entries
  double* ddiag = h->d_rhs.p + n + 64;
  double* dd = ddiag + n;
  double* beta = dd + n;        // q = alpha / d, then K^-1 q in place
  double* cw = beta + n;
  // pass 1: alpha and d = diag(K^-1), K^-1 resident as in bgp_dense_grad_terms
  BGP_CUDA(cudaMemcpyAsync(alpha, r, sizeof(double) * n, cudaMemcpyHostToDevice, s));
  BGP_TRY(dense_potrs_dev(h, alpha, 1, n));
  BGP_TRY(h->d_inv.reserve((size_t)n * n, s));
  BGP_TRY(fill_identity_launch(h->d_inv.p, n, s));
  BGP_TRY(dense_potrs_dev(h, h->d_inv.p, n, n));
  BGP_TRY(slab_diag_launch(h->d_inv.p, n, 0, n, dd, s));
  std::vector<double> d_host((size_t)n);
  if (alpha_out) BGP_CUDA(cudaMemcpyAsync(alpha_out, alpha, sizeof(double) * n, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaMemcpyAsync(d_host.data(), dd, sizeof(double) * n, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  if (d_out) memcpy(d_out, d_host.data(), sizeof(double) * n);
  if (!grad) return BGP_OK;
  BGP_TRY(loo_check_diag(d_host.data(), n));
  // pass 2: beta = K^-1 (alpha / d); G = diag(sqrt(c)) K^-1 in place; A = -(G^T G) (lower, mirrored) on the tensor pipe,
  // plus 1/2 (beta alpha^T + alpha beta^T); then the contraction of bgp_kmat_gradient_contract (A given whole)
  BGP_TRY(loo_weights_launch(alpha, dd, n, beta, cw, s));
  BGP_TRY(dense_potrs_dev(h, beta, 1, n));
  BGP_TRY(scale_rows_launch(h->d_inv.p, n, n, n, cw, true, s));
  DevBuf<double> dA, slices;
  DevBuf<GemmDesc> descs;
  BGP_TRY(dA.alloc((size_t)n * n, s));
  BGP_CUDA(cudaMemsetAsync(dA.p, 0, sizeof(double) * n * n, s));
  BGP_TRY(predict_gemm_sub(h->d_inv.p, n, h->d_inv.p, n, n, n, n, true, dA.p, n, slices, descs, s));
  slices.release();
  BGP_TRY(loo_form_a_members(dA.p, n, alpha, beta, 1, s));
  BGP_TRY(h->d_which.reserve(std::max(np, 1), s));
  if (np) BGP_CUDA(cudaMemcpyAsync(h->d_which.p, which, sizeof(unsigned) * np, cudaMemcpyHostToDevice, s));
  BGP_TRY(kmat_grad_contract_launch(h->d_prog.p, h->ndim, np, h->d_which.p, h->d_x.p, n, dA.p, n, nullptr, 0.0, 1.0, dg,
                                    diag_out ? ddiag : nullptr, h->d_gscratch, s));
  if (beta_out) BGP_CUDA(cudaMemcpyAsync(beta_out, beta, sizeof(double) * n, cudaMemcpyDeviceToHost, s));
  if (np && g_out) BGP_CUDA(cudaMemcpyAsync(g_out, dg, sizeof(double) * np, cudaMemcpyDeviceToHost, s));
  if (diag_out) BGP_CUDA(cudaMemcpyAsync(diag_out, ddiag, sizeof(double) * n, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  return BGP_OK;
}

int bgp_dense_predict(bgp_dense_t* h, const bgp_kernel_spec_t* spec, const double* xs, int64_t ns, int32_t what,
                      double* out) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  if (!h->has_inputs) { set_error("the factor was imported: the handle holds no kernel/coordinates"); return BGP_ERR_NOT_COMPUTED; }
  if (what != BGP_PREDICT_VAR && what != BGP_PREDICT_COV) { set_error("invalid prediction kind %d", what); return BGP_ERR_INVALID; }
  if (ns < 0) { set_error("negative number of test points"); return BGP_ERR_INVALID; }
  DevProgram P;
  BGP_TRY(build_dev_program(spec, &P));
  if (P.ndim != h->ndim) { set_error("dimension mismatch: kernel ndim %d, input ndim %d", P.ndim, h->ndim); return BGP_ERR_DIM; }
  if (ns == 0) return BGP_OK;
  const int64_t n = h->n;
  const int nd = h->ndim;
  cudaStream_t s = h->s;
  DevBuf<DevProgram> dprog;
  DevBuf<double> dxs, dW, dkd, dvar, dC, scratch;
  if (what == BGP_PREDICT_VAR) {
    BGP_TRY(upload_program(P, dprog, s));
    const int64_t c = std::min(ns, predict_chunk_cols(n, 1));
    // workspace n*c + O(c): var_j = k(x*_j, x*_j) - ||L^-1 K(x, x*_j)||^2, chunk by chunk
    BGP_TRY(dxs.alloc((size_t)c * nd, s));
    BGP_TRY(dW.alloc((size_t)n * c, s));
    BGP_TRY(dkd.alloc((size_t)c, s));
    BGP_TRY(dvar.alloc((size_t)c, s));
    for (int64_t j0 = 0; j0 < ns; j0 += c) {
      const int64_t nc = std::min(c, ns - j0);
      BGP_CUDA(cudaMemcpyAsync(dxs.p, xs + j0 * nd, sizeof(double) * nc * nd, cudaMemcpyHostToDevice, s));
      BGP_TRY(kmat_general_launch_auto(P, dprog.p, dxs.p, nc, h->d_x.p, n, dW.p, n, s));  // K(x, x*_chunk), N x nc
      BGP_TRY(dense_trsm_fwd_dev(h, dW.p, nc, n));
      BGP_TRY(kmat_diagonal_launch(dprog.p, dxs.p, dxs.p, nc, dkd.p, s));
      BGP_TRY(predict_var_launch(dW.p, n, dW.p, n, n, nc, dkd.p, dvar.p, scratch, s));
      BGP_CUDA(cudaMemcpyAsync(out + j0, dvar.p, sizeof(double) * nc, cudaMemcpyDeviceToHost, s));
    }
  } else {
    BGP_TRY(dense_predict_cov_dev(h, P, xs, ns, dC));
    BGP_CUDA(cudaMemcpyAsync(out, dC.p, sizeof(double) * ns * ns, cudaMemcpyDeviceToHost, s));
  }
  BGP_CUDA(cudaStreamSynchronize(s));
  return BGP_OK;
}

// GP.grad_predict's var and dvar: bgp_dense_predict's VAR chunks, then per chunk W <- L^-T W (= K^-1 K(x, x*_chunk))
// in place and dvar = dprior - 2 sum_j d1 k(x*, x_j) W_j (kmat_x1_grad_matvec_launch)
int bgp_dense_predict_grad(bgp_dense_t* h, const bgp_kernel_spec_t* spec, const double* xs, int64_t ns, double* var,
                           double* dvar) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  if (!h->has_inputs) { set_error("the factor was imported: the handle holds no kernel/coordinates"); return BGP_ERR_NOT_COMPUTED; }
  if (ns < 0) { set_error("negative number of test points"); return BGP_ERR_INVALID; }
  DevProgram P;
  BGP_TRY(build_dev_program(spec, &P));
  if (P.ndim != h->ndim) { set_error("dimension mismatch: kernel ndim %d, input ndim %d", P.ndim, h->ndim); return BGP_ERR_DIM; }
  if (P.ndim > BGP_MAX_DIM) { set_error("input-coordinate gradients support at most %d dimensions (got %d)", BGP_MAX_DIM, P.ndim); return BGP_ERR_INVALID; }
  if (ns == 0) return BGP_OK;
  const int64_t n = h->n;
  const int nd = h->ndim;
  cudaStream_t s = h->s;
  DevBuf<DevProgram> dprog;
  DevBuf<double> dxs, dW, dkd, dvar_c, ddvar, scratch;
  BGP_TRY(upload_program(P, dprog, s));
  const int64_t c = std::min(ns, predict_chunk_cols(n, 1));
  // workspace n*c + O(c * ndim): bgp_dense_predict's VAR workspace plus the chunk's dvar
  BGP_TRY(dxs.alloc((size_t)c * nd, s));
  BGP_TRY(dW.alloc((size_t)n * c, s));
  BGP_TRY(dkd.alloc((size_t)c, s));
  BGP_TRY(dvar_c.alloc((size_t)c, s));
  BGP_TRY(ddvar.alloc((size_t)c * nd, s));
  for (int64_t j0 = 0; j0 < ns; j0 += c) {
    const int64_t nc = std::min(c, ns - j0);
    // the steps of bgp_dense_predict's VAR loop
    BGP_CUDA(cudaMemcpyAsync(dxs.p, xs + j0 * nd, sizeof(double) * nc * nd, cudaMemcpyHostToDevice, s));
    BGP_TRY(kmat_general_launch_auto(P, dprog.p, dxs.p, nc, h->d_x.p, n, dW.p, n, s));
    BGP_TRY(dense_trsm_fwd_dev(h, dW.p, nc, n));
    BGP_TRY(kmat_diagonal_launch(dprog.p, dxs.p, dxs.p, nc, dkd.p, s));
    BGP_TRY(predict_var_launch(dW.p, n, dW.p, n, n, nc, dkd.p, dvar_c.p, scratch, s));
    BGP_CUDA(cudaMemcpyAsync(var + j0, dvar_c.p, sizeof(double) * nc, cudaMemcpyDeviceToHost, s));
    BGP_TRY(dense_trsm_bwd_dev(h, dW.p, nc, n));
    BGP_TRY(kmat_x1_grad_matvec_launch(P, dprog.p, dxs.p, nc, h->d_x.p, n, dW.p, n, -2.0, 1, ddvar.p, scratch, s));
    BGP_CUDA(cudaMemcpyAsync(dvar + j0 * nd, ddvar.p, sizeof(double) * nc * nd, cudaMemcpyDeviceToHost, s));
  }
  BGP_CUDA(cudaStreamSynchronize(s));
  return BGP_OK;
}

int bgp_dense_sample(bgp_dense_t* h, const bgp_kernel_spec_t* spec, const double* xs, int64_t ns, const double* mean,
                     const double* z, int64_t size, double jitter, double* out) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  if (!h->has_inputs) { set_error("the factor was imported: the handle holds no kernel/coordinates"); return BGP_ERR_NOT_COMPUTED; }
  BGP_TRY(mvn_sample_check(ns, size, jitter));
  DevProgram P;
  BGP_TRY(build_dev_program(spec, &P));
  if (P.ndim != h->ndim) { set_error("dimension mismatch: kernel ndim %d, input ndim %d", P.ndim, h->ndim); return BGP_ERR_DIM; }
  if (ns == 0 || size == 0) return BGP_OK;
  DevBuf<double> dC;
  BGP_TRY(sample_mark(0, h->s));
  BGP_TRY(dense_predict_cov_dev(h, P, xs, ns, dC));
  return mvn_draw_host_io(dC.p, ns, mean, z, size, jitter, out, h->s);
}

int bgp_dense_export_factor(bgp_dense_t* h, double* out) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  const int64_t n = h->n;
  BGP_CUDA(cudaMemcpyAsync(out, h->d_A.p, sizeof(double) * n * n, cudaMemcpyDeviceToHost, h->s));
  BGP_CUDA(cudaStreamSynchronize(h->s));
  for (int64_t j = 1; j < n; ++j)
    for (int64_t i = 0; i < j; ++i) out[j * n + i] = 0.0;  // column-major: element (i, j) with i < j
  return BGP_OK;
}

int bgp_dense_import_factor(bgp_dense_t* h, const double* factor, int64_t n, double log_det) {
  if (!h || n <= 0) { set_error("invalid argument"); return BGP_ERR_INVALID; }
  h->computed = false;
  BGP_TRY(require_device());
  if (!h->s) {
    BGP_CUDA(cudaStreamCreateWithFlags(&h->s, cudaStreamNonBlocking));
    for (int i = 0; i < 4; ++i) BGP_CUDA(cudaEventCreate(&h->ev[i]));
  }
  h->n = n;
  h->has_inputs = false;
  BGP_TRY(h->d_A.reserve((size_t)n * n, h->s));
  BGP_TRY(h->d_scalar.reserve(2, h->s));
  BGP_CUDA(cudaMemcpyAsync(h->d_A.p, factor, sizeof(double) * n * n, cudaMemcpyHostToDevice, h->s));
  BGP_CUDA(cudaStreamSynchronize(h->s));
  h->log_det = log_det;
  h->computed = true;
  return BGP_OK;
}

int bgp_dense_last_timing(const bgp_dense_t* h, double* ms2) {
  if (!h) { set_error("null handle"); return BGP_ERR_INVALID; }
  ms2[0] = h->t_ms[0]; ms2[1] = h->t_ms[1];
  return BGP_OK;
}

}  // extern "C"

// ---- batched log-likelihood terms and predictions: many parameter vectors of one kernel program on the same x -------
// The stream is a base so that it is destroyed after the buffers: each DevBuf destructor issues its cudaFreeAsync on
// it, then the stream is synchronised and destroyed.
struct BatchStream {
  cudaStream_t s = nullptr;
  ~BatchStream() {
    if (s) {
      cudaStreamSynchronize(s);
      cudaStreamDestroy(s);
    }
  }
};
struct bgp_dense_batch : BatchStream {
  DevBuf<DevProgram> d_prog;
  DevBuf<double> d_x, d_yerr, d_diag, d_r, d_sol, d_tmp, d_A, d_out, d_fn;
  DevBuf<int> d_info;
  DevBuf<GemmDesc> d_gdesc;
  // bgp_dense_batch_predict: test points, the member means and their matvec partials, W = L^-1 K(x, x*), k(x*, x*),
  // variances and their partials, covariances and their split-K slices
  DevBuf<double> d_xs, d_mean, d_mvp, d_W, d_kd, d_var, d_vp, d_C, d_slices;
  DevBuf<GemmDesc> d_pdesc;
  // bgp_dense_batch_sample: the means, normals and draws, the covariance factorisations' info words and the product's
  // descriptors (apart from d_gdesc, which the factorisations use)
  DevBuf<double> d_madd, d_z, d_draws;
  DevBuf<int> d_dinfo;
  DevBuf<GemmDesc> d_sdesc;
  // bgp_dense_batch_grad_terms: K_b^-1, the contraction partials and g
  DevBuf<double> d_inv, d_gp, d_g;
  DevBuf<unsigned> d_which;
  // bgp_dense_batch_predict_grad: dmu, a test-point chunk of dvar and the input-gradient contraction's partials
  DevBuf<double> d_dmu, d_dvar, d_xgp;
  // bgp_dense_batch_loo_terms (besides d_inv, d_gp, d_g and d_which): A, beta (q, then K^-1 q) and c
  DevBuf<double> d_loo_a, d_beta, d_cw;
  // bgp_dense_batch_fisher_terms (besides d_inv, d_gp, d_g, d_which and d_slices): the plane / product buffer P, T,
  // the rows and their diagonals, the white-noise vectors and the mean gradients (K^-1 dmu^T after the solve)
  DevBuf<double> d_fp, d_ft, d_frows, d_frd, d_fv, d_fdmu;
};

// members per chunk: as many members of per_member doubles as fit in 4 GiB, at least one; BGP_BATCH_CHUNK=<members>
// overrides it (read at every call, so that tests can force several chunks and a ragged tail at small n)
static int64_t batch_chunk_members(int64_t per_member, int64_t B) {
  int64_t c = std::max<int64_t>(1, (int64_t(4) << 30) / (per_member * (int64_t)sizeof(double)));
  if (const char* e = getenv("BGP_BATCH_CHUNK")) {
    const long v = atol(e);
    if (v >= 1) c = v;
  }
  return std::min<int64_t>(std::min<int64_t>(c, B), 65535);  // grid.y / grid.z carry the member index
}

// member spec = template with the parameter slots of each leaf, in node order, replaced by p: the leaf's own
// parameters (params[0 .. n_params)) followed by its metric (metric[0 .. n_metric)), at the offsets the template's
// program assigns (DevLeaf::param_off, the order of bgp_spec_num_params)
static void patch_member_spec(const bgp_kernel_spec_t* tmpl, const DevProgram& Pt, const double* p,
                              bgp_kernel_spec_t* out) {
  *out = *tmpl;
  int l = 0;
  for (int i = 0; i < tmpl->n_nodes; ++i) {
    bgp_kernel_node_t& k = out->nodes[i];
    if (k.op != BGP_OP_KERNEL) continue;
    const DevLeaf& L = Pt.leaf[l++];
    for (int j = 0; j < L.n_params; ++j) k.params[j] = p[L.param_off + j];
    for (int j = 0; j < L.n_metric; ++j) k.metric[j] = p[L.param_off + L.n_params + j];
  }
}

// The start of every batched entry point: the argument checks, then (B > 0) one program per member built on the host
// and uploaded with x.  A member whose program fails validation evaluates the template's program in its slot (reported
// as info = -1, its results are discarded).
struct BatchPrograms {
  std::vector<DevProgram> progs;
  std::vector<char> valid;
};
static int batch_begin(bgp_dense_batch* h, const bgp_kernel_spec_t* spec, const double* params, int64_t B, int64_t P,
                       const double* x, int64_t n, int32_t ndim, BatchPrograms* bp) {
  if (!h) { set_error("null handle"); return BGP_ERR_INVALID; }
  if (n <= 0) { set_error("invalid number of points"); return BGP_ERR_INVALID; }
  if (B < 0) { set_error("negative number of parameter vectors"); return BGP_ERR_INVALID; }
  DevProgram Pt;
  BGP_TRY(build_dev_program(spec, &Pt));
  if (P != Pt.n_params_total) {
    set_error("the program has %d parameters, the parameter matrix %lld columns", Pt.n_params_total, (long long)P);
    return BGP_ERR_INVALID;
  }
  if (Pt.ndim != ndim) { set_error("dimension mismatch: kernel ndim %d, input ndim %d", Pt.ndim, ndim); return BGP_ERR_DIM; }
  if (B == 0) return BGP_OK;
  BGP_TRY(require_device());
  if (!h->s) BGP_CUDA(cudaStreamCreateWithFlags(&h->s, cudaStreamNonBlocking));
  bp->progs.assign((size_t)B, DevProgram());
  bp->valid.assign((size_t)B, 1);
  bgp_kernel_spec_t ms;
  for (int64_t b = 0; b < B; ++b) {
    patch_member_spec(spec, Pt, params + b * P, &ms);
    if (build_dev_program(&ms, &bp->progs[b]) != BGP_OK || bp->progs[b].ndim != ndim) { bp->valid[b] = 0; bp->progs[b] = Pt; }
  }
  return BGP_OK;
}

// the shared buffers of a chunk of `chunk` members (d_A is reserved by the caller) and the programs and x of all B
static int batch_reserve_common(bgp_dense_batch* h, const BatchPrograms& bp, const double* x, int64_t n, int32_t ndim,
                                int64_t chunk, int64_t tmp_cols) {
  cudaStream_t s = h->s;
  const int64_t B = (int64_t)bp.progs.size();
  BGP_TRY(h->d_prog.reserve((size_t)B, s));
  BGP_TRY(h->d_x.reserve((size_t)n * ndim, s));
  BGP_TRY(h->d_yerr.reserve((size_t)n * chunk, s));
  BGP_TRY(h->d_diag.reserve((size_t)n * chunk, s));
  BGP_TRY(h->d_r.reserve((size_t)n * chunk, s));
  BGP_TRY(h->d_sol.reserve((size_t)n * chunk, s));
  BGP_TRY(h->d_tmp.reserve((size_t)n * chunk * tmp_cols, s));
  BGP_TRY(h->d_info.reserve((size_t)chunk, s));
  BGP_CUDA(cudaMemcpyAsync(h->d_prog.p, bp.progs.data(), sizeof(DevProgram) * B, cudaMemcpyHostToDevice, s));
  BGP_CUDA(cudaMemcpyAsync(h->d_x.p, x, sizeof(double) * n * ndim, cudaMemcpyHostToDevice, s));
  return BGP_OK;
}

// the test points of the predictive entry points in d_xs (at least one double)
static int batch_upload_xs(bgp_dense_batch* h, const double* xs, int64_t ns, int32_t ndim) {
  BGP_TRY(h->d_xs.reserve((size_t)std::max<int64_t>(1, ns * ndim), h->s));
  if (ns > 0) BGP_CUDA(cudaMemcpyAsync(h->d_xs.p, xs, sizeof(double) * ns * ndim, cudaMemcpyHostToDevice, h->s));
  return BGP_OK;
}

// members [c0, c0 + mc): K_b + diag(yerr_b^2) built and factorised in place (d_A, member stride n^2, info in d_info) and
// alpha_b = K_b^-1 r_b in d_sol (member stride n): the steps of bgp_dense_compute and of the few-right-hand-side solve
// of bgp_dense_apply_inverse / bgp_dense_dot_solve, member-indexed, one launch per step for the whole chunk.  A NULL r
// (bgp_dense_batch_fisher_terms without residuals) skips the residual upload and the alpha solve.
static int batch_factor_chunk(bgp_dense_batch* h, const BatchPrograms& bp, int64_t c0, int mc, int64_t n,
                              const double* yerr, const double* r) {
  cudaStream_t s = h->s;
  const int64_t len = (int64_t)mc * n;
  const int64_t mstride = n * n;
  BGP_CUDA(cudaMemcpyAsync(h->d_yerr.p, yerr + c0 * n, sizeof(double) * len, cudaMemcpyHostToDevice, s));
  if (r) BGP_CUDA(cudaMemcpyAsync(h->d_r.p, r + c0 * n, sizeof(double) * len, cudaMemcpyHostToDevice, s));
  BGP_CUDA(cudaMemsetAsync(h->d_info.p, 0, sizeof(int) * mc, s));
  // yerr^2 exactly as bgp_dense_compute squares it (an elementwise product: the layout does not matter)
  square2_kernel<<<(unsigned)std::min<int64_t>((len + 255) / 256, 1184), 256, 0, s>>>(h->d_yerr.p, h->d_diag.p, len);
  BGP_LAUNCH_CHECK();
  BGP_TRY(kmat_symmetric_batch_launch_auto(bp.progs.data() + c0, h->d_prog.p + c0, mc, h->d_x.p, n, h->d_diag.p,
                                           h->d_A.p, mstride, h->d_fn, s));
  BGP_TRY(dense_potrf_members(h->d_A.p, n, mstride, mc, h->d_info.p, nullptr, h->d_gdesc, s));
  if (!r) return BGP_OK;
  BGP_CUDA(cudaMemcpyAsync(h->d_sol.p, h->d_r.p, sizeof(double) * len, cudaMemcpyDeviceToDevice, s));
  return potrs_small_members(h->d_A.p, n, h->d_sol.p, 1, n, h->d_tmp.p, mc, mstride, n, s);
}

// a device buffer of a member chunk: `per` doubles per member, at least one double in all
struct ChunkBuf {
  DevBuf<double>* buf;
  int64_t per;
};
// a host output of a batched entry point: member b's row of `len` doubles at p + b * len (p may be null)
struct BatchOut {
  double* p;
  int64_t len;
};

// The member chunking of every batched entry point, after batch_begin with B > 0.  A chunk has as many members as
// the per-member workspace allows (batch_chunk_members), at most `cap` (one launch's descriptors), halved while the
// chunk buffers `bufs` do not fit (BGP_ERR_NOMEM when one member's do not); then come the shared buffers and
// setup(chunk), the entry point's own.  Each chunk of mc members from c0 runs batch_factor_chunk, then step(c0, mc,
// progs, dprogs) with the members' host and device programs, copies the info words and synchronises.  Last, a member
// whose program failed validation gets info = -1, and every output row of a member with info != 0 is NaN.
template <class Setup, class Step>
static int batch_run(bgp_dense_batch* h, const BatchPrograms& bp, const double* x, int64_t n, int32_t ndim,
                     const double* yerr, const double* r, int64_t per_member, int64_t cap, int64_t tmp_cols,
                     const std::vector<ChunkBuf>& bufs, Setup setup, Step step, int32_t* info,
                     std::initializer_list<BatchOut> outs) {
  cudaStream_t s = h->s;
  const int64_t B = (int64_t)bp.progs.size();
  int64_t chunk = std::max<int64_t>(1, std::min(batch_chunk_members(per_member, B), cap));
  for (;;) {
    int st = BGP_OK;
    for (const ChunkBuf& b : bufs)
      if ((st = b.buf->reserve((size_t)std::max<int64_t>(1, b.per * chunk), s)) != BGP_OK) break;
    if (st == BGP_OK) break;
    if (st != BGP_ERR_NOMEM || chunk == 1) return st;
    for (const ChunkBuf& b : bufs) b.buf->release();
    chunk = (chunk + 1) / 2;
  }
  BGP_TRY(batch_reserve_common(h, bp, x, n, ndim, chunk, tmp_cols));
  BGP_TRY(setup(chunk));
  for (int64_t c0 = 0; c0 < B; c0 += chunk) {
    const int mc = (int)std::min(chunk, B - c0);
    BGP_TRY(batch_factor_chunk(h, bp, c0, mc, n, yerr, r));
    BGP_TRY(step(c0, mc, bp.progs.data() + c0, h->d_prog.p + c0));
    BGP_CUDA(cudaMemcpyAsync(info + c0, h->d_info.p, sizeof(int) * mc, cudaMemcpyDeviceToHost, s));
    BGP_CUDA(cudaStreamSynchronize(s));
  }
  for (int64_t b = 0; b < B; ++b) {
    if (!bp.valid[b]) info[b] = -1;
    if (info[b] == 0) continue;
    for (const BatchOut& o : outs)
      if (o.p) std::fill(o.p + b * o.len, o.p + (b + 1) * o.len, std::nan(""));
  }
  return BGP_OK;
}

// The test-point chunking of the predictive entry points: chunks of c test points (the single path's
// predict_chunk_cols(n, 1), whatever the number of members) ending in a ragged tail, the mean matvec's partials per
// member, a VAR chunk's partials (var) and the split-K plan of the COV product (cov)
struct BatchTestPlan {
  int64_t c, tail, mvp, vp = 0, gsplit = 1;
  BatchTestPlan(int64_t n, int64_t ns, bool var, bool cov)
      : c(std::min(ns, predict_chunk_cols(n, 1))), tail(c > 0 ? ns - (ns - 1) / c * c : 0),
        mvp(matvec_partial_size(ns, n)) {
    if (var) vp = std::max(predict_var_partial_size(n, c), predict_var_partial_size(n, tail));
    int64_t gklen = 0;
    if (cov && ns > 0) predict_gemm_plan(ns, ns, n, &gsplit, &gklen);
  }
};

// members [0, mc) after batch_factor_chunk: log_det_b into d_out and quad_b = r_b^T K_b^-1 r_b, a fixed-order dot of
// r_b and alpha_b, into d_out + chunk
static int batch_loglik_chunk(bgp_dense_batch* h, int mc, int64_t n, int64_t chunk) {
  logdet_diag_kernel<<<(unsigned)mc, 1024, 0, h->s>>>(h->d_A.p, n, n, h->d_out.p, n * n);
  BGP_LAUNCH_CHECK();
  dot_rows_kernel<<<(unsigned)mc, 256, 0, h->s>>>(h->d_r.p, h->d_sol.p, n, h->d_out.p + chunk);
  BGP_LAUNCH_CHECK();
  return BGP_OK;
}

// members [0, mc) after batch_factor_chunk: mean_b = K_b(x*, x) alpha_b into d_mean (member stride ns), the matvec
// GP.predict computes for its mean
static int batch_mean_chunk(bgp_dense_batch* h, const DevProgram* dprogs, int32_t ndim, int mc, int64_t n, int64_t ns) {
  return kmat_matvec_batch_launch(dprogs, ndim, mc, h->d_xs.p, ns, h->d_x.p, n, h->d_sol.p, n, h->d_mean.p, ns,
                                  h->d_mvp.p, h->s);
}

// members [0, mc) after batch_factor_chunk, test points [j0, j0 + nc) of a VAR chunk of c: the steps of
// bgp_dense_predict's variance loop, member-indexed.  W = L_b^-1 K_b(x, x*) (d_W, the columns of all members
// interleaved as in batch_cov_chunk), k(x*, x*) and the variances (d_var, member stride c), copied to var + j0 on the
// host (member stride ns).
static int batch_var_chunk(bgp_dense_batch* h, const DevProgram* progs, const DevProgram* dprogs, int mc, int64_t n,
                           int32_t ndim, int64_t c, int64_t j0, int64_t nc, double* var, int64_t ns) {
  cudaStream_t s = h->s;
  const int64_t ldw = (int64_t)mc * n;
  const double* xc = h->d_xs.p + j0 * ndim;
  BGP_TRY(kmat_general_batch_launch_auto(progs, dprogs, mc, xc, nc, h->d_x.p, n, h->d_W.p, ldw, n, h->d_fn, s));
  BGP_TRY(trsm_fwd_members(h->d_A.p, n, n * n, h->d_W.p, nc, ldw, n, mc, h->d_tmp.p, ldw, s));
  BGP_TRY(kmat_diagonal_launch(dprogs, xc, xc, nc, h->d_kd.p, s, mc, c));
  BGP_TRY(predict_var_batch_launch(h->d_W.p, ldw, h->d_W.p, ldw, n, nc, h->d_kd.p, h->d_var.p, mc, n, c, h->d_vp, s));
  BGP_CUDA(cudaMemcpy2DAsync(var + j0, sizeof(double) * ns, h->d_var.p, sizeof(double) * c, sizeof(double) * nc, mc,
                             cudaMemcpyDeviceToHost, s));
  return BGP_OK;
}

// members [0, mc) after batch_factor_chunk: the steps of bgp_dense_predict's covariance path, member-indexed:
// K**, every W chunk resident (W = L_b^-1 K_b(x, x*), test-point chunks of c columns), C_b = K** - W^T W into d_C
// (member stride ns^2).  The W columns of all members are interleaved: column j of member m at W + (j * mc + m) * n, so
// that the columns of a test-point chunk are one contiguous block (the few-column solve copies its result back in one
// piece).  bgp_dense_batch_predict copies C out; bgp_dense_batch_sample draws from it on the device.
static int batch_cov_chunk(bgp_dense_batch* h, const DevProgram* progs, const DevProgram* dprogs, int mc, int64_t n,
                           int32_t ndim, int64_t ns, int64_t c) {
  cudaStream_t s = h->s;
  const int64_t nn = n * n, ldw = (int64_t)mc * n;
  BGP_TRY(kmat_symmetric_batch_launch_auto(progs, dprogs, mc, h->d_xs.p, ns, nullptr, h->d_C.p, ns * ns, h->d_fn, s));
  for (int64_t j0 = 0; j0 < ns; j0 += c) {
    const int64_t nc = std::min(c, ns - j0);
    BGP_TRY(kmat_general_batch_launch_auto(progs, dprogs, mc, h->d_xs.p + j0 * ndim, nc, h->d_x.p, n,
                                           h->d_W.p + j0 * ldw, ldw, n, h->d_fn, s));
    BGP_TRY(trsm_fwd_members(h->d_A.p, n, nn, h->d_W.p + j0 * ldw, nc, ldw, n, mc, h->d_tmp.p, ldw, s));
  }
  return predict_gemm_sub_members(h->d_W.p, ldw, h->d_W.p, ldw, ns, ns, n, true, h->d_C.p, ns, mc, n, ns * ns,
                                  h->d_slices, h->d_pdesc, s);
}

extern "C" {

int bgp_dense_batch_create(bgp_dense_batch_t** out) {
  *out = new (std::nothrow) bgp_dense_batch();
  if (!*out) { set_error("out of host memory"); return BGP_ERR_NOMEM; }
  return BGP_OK;
}

void bgp_dense_batch_destroy(bgp_dense_batch_t* h) { delete h; }

int bgp_dense_batch_log_likelihood(bgp_dense_batch_t* h, const bgp_kernel_spec_t* spec, const double* params,
                                   int64_t B, int64_t P, const double* x, int64_t n, int32_t ndim,
                                   const double* yerr, const double* r,
                                   double* log_det, double* quad, int32_t* info) {
  BatchPrograms bp;
  BGP_TRY(batch_begin(h, spec, params, B, P, x, n, ndim, &bp));
  if (B == 0) return BGP_OK;
  cudaStream_t s = h->s;
  const int64_t nn = n * n;
  int64_t chunk = 0;
  auto setup = [&](int64_t c) {
    chunk = c;
    return h->d_out.reserve((size_t)2 * c, s);
  };
  auto step = [&](int64_t c0, int mc, const DevProgram*, const DevProgram*) -> int {
    BGP_TRY(batch_loglik_chunk(h, mc, n, chunk));
    BGP_CUDA(cudaMemcpyAsync(log_det + c0, h->d_out.p, sizeof(double) * mc, cudaMemcpyDeviceToHost, s));
    BGP_CUDA(cudaMemcpyAsync(quad + c0, h->d_out.p + chunk, sizeof(double) * mc, cudaMemcpyDeviceToHost, s));
    return BGP_OK;
  };
  return batch_run(h, bp, x, n, ndim, yerr, r, nn, 65535, 1, {{&h->d_A, nn}}, setup, step, info,
                   {{log_det, 1}, {quad, 1}});
}

int bgp_dense_batch_grad_terms(bgp_dense_batch_t* h, const bgp_kernel_spec_t* spec, const double* params, int64_t B,
                               int64_t P, const double* x, int64_t n, int32_t ndim, const double* yerr, const double* r,
                               const uint32_t* which, double* log_det, double* quad, double* alpha, double* diag,
                               double* g, int32_t* info) {
  if (P > 64) { set_error("gradient supports at most 64 hyper-parameters"); return BGP_ERR_INVALID; }
  BatchPrograms bp;
  BGP_TRY(batch_begin(h, spec, params, B, P, x, n, ndim, &bp));
  if (B == 0) return BGP_OK;
  cudaStream_t s = h->s;
  const int64_t nn = n * n;
  // n <= DS_MAX_RHS: K^-1 goes through the few-column solve, as bgp_dense_grad_terms sends it, with n x n of scratch
  const int64_t tmp_cols = n <= DS_MAX_RHS ? n : 1;
  const int64_t nt = (n + 31) / 32;  // the contraction's 32 x 32 tiles
  // doubles per member (see include/bgp.h): factor, K^-1, the vectors of batch_reserve_common, partials, g
  const int64_t per_member = 2 * nn + (4 + tmp_cols) * n + nt * nt * P + P;
  int64_t chunk = 0;
  auto setup = [&](int64_t c) -> int {
    chunk = c;
    BGP_TRY(h->d_out.reserve((size_t)2 * c, s));
    BGP_TRY(h->d_which.reserve((size_t)std::max<int64_t>(1, P), s));
    if (P > 0) BGP_CUDA(cudaMemcpyAsync(h->d_which.p, which, sizeof(unsigned) * P, cudaMemcpyHostToDevice, s));
    return BGP_OK;
  };
  // the steps of bgp_dense_compute and bgp_dense_grad_terms, member-indexed: log_det and quad as
  // bgp_dense_batch_log_likelihood computes them
  auto step = [&](int64_t c0, int mc, const DevProgram*, const DevProgram* dprogs) -> int {
    BGP_TRY(batch_loglik_chunk(h, mc, n, chunk));
    // K_b^-1 by solving against the identity
    BGP_TRY(fill_identity_members(h->d_inv.p, n, mc, s));
    BGP_TRY(potrs_members(h->d_A.p, n, nn, h->d_inv.p, n, n, nn, mc, h->d_tmp.p, s));
    // g_b and diag(alpha_b alpha_b^T - K_b^-1); the diagonal goes to d_diag, whose yerr^2 the build above consumed
    BGP_TRY(kmat_grad_contract_members(dprogs, (int)P, h->d_which.p, h->d_x.p, n, h->d_inv.p, n, nn, h->d_sol.p, n,
                                       1.0, -1.0, h->d_g.p, P, diag ? h->d_diag.p : nullptr, n, mc, h->d_gp, s));
    if (log_det) BGP_CUDA(cudaMemcpyAsync(log_det + c0, h->d_out.p, sizeof(double) * mc, cudaMemcpyDeviceToHost, s));
    if (quad) BGP_CUDA(cudaMemcpyAsync(quad + c0, h->d_out.p + chunk, sizeof(double) * mc, cudaMemcpyDeviceToHost, s));
    if (alpha) BGP_CUDA(cudaMemcpyAsync(alpha + c0 * n, h->d_sol.p, sizeof(double) * mc * n, cudaMemcpyDeviceToHost, s));
    if (diag) BGP_CUDA(cudaMemcpyAsync(diag + c0 * n, h->d_diag.p, sizeof(double) * mc * n, cudaMemcpyDeviceToHost, s));
    if (g && P > 0) BGP_CUDA(cudaMemcpyAsync(g + c0 * P, h->d_g.p, sizeof(double) * mc * P, cudaMemcpyDeviceToHost, s));
    return BGP_OK;
  };
  return batch_run(h, bp, x, n, ndim, yerr, r, per_member, 65535, tmp_cols,
                   {{&h->d_A, nn}, {&h->d_inv, nn}, {&h->d_gp, nt * nt * P}, {&h->d_g, P}}, setup, step, info,
                   {{log_det, 1}, {quad, 1}, {alpha, n}, {diag, n}, {g, P}});
}

int bgp_dense_batch_loo_terms(bgp_dense_batch_t* h, const bgp_kernel_spec_t* spec, const double* params, int64_t B,
                              int64_t P, const double* x, int64_t n, int32_t ndim, const double* yerr, const double* r,
                              const uint32_t* which, double* alpha, double* d, double* beta, double* g, double* diag,
                              int32_t* info) {
  const bool grad = which != nullptr;
  if (grad && P > 64) { set_error("gradient supports at most 64 hyper-parameters"); return BGP_ERR_INVALID; }
  BatchPrograms bp;
  BGP_TRY(batch_begin(h, spec, params, B, P, x, n, ndim, &bp));
  if (B == 0) return BGP_OK;
  cudaStream_t s = h->s;
  const int64_t nn = n * n;
  // n <= DS_MAX_RHS: K^-1 goes through the few-column solve, as bgp_dense_loo_terms sends it, with n x n of scratch
  const int64_t tmp_cols = n <= DS_MAX_RHS ? n : 1;
  const int64_t nt = (n + 31) / 32;  // the contraction's 32 x 32 tiles
  // the G^T G product's split-K plan, bgp_dense_loo_terms' (no slice buffer with one slice)
  int64_t gsplit = 1, gklen = 0;
  if (grad) predict_gemm_plan(n, n, n, &gsplit, &gklen);
  const int64_t slices = gsplit > 1 ? gsplit * nn : 0;
  // doubles per member (see include/bgp.h): factor, K^-1 and the vectors of batch_reserve_common; pass 2 adds A, the
  // product's slices, beta, c, the contraction partials and g
  int64_t per_member = 2 * nn + (4 + tmp_cols) * n;
  std::vector<ChunkBuf> bufs = {{&h->d_A, nn}, {&h->d_inv, nn}};
  if (grad) {
    per_member += nn + slices + 2 * n + nt * nt * P + P;
    bufs.insert(bufs.end(), {{&h->d_loo_a, nn}, {&h->d_slices, slices}, {&h->d_beta, n}, {&h->d_cw, n},
                             {&h->d_gp, nt * nt * P}, {&h->d_g, P}});
  }
  auto setup = [&](int64_t) -> int {
    if (!grad) return BGP_OK;
    BGP_TRY(h->d_which.reserve((size_t)std::max<int64_t>(1, P), s));
    if (P > 0) BGP_CUDA(cudaMemcpyAsync(h->d_which.p, which, sizeof(unsigned) * P, cudaMemcpyHostToDevice, s));
    return BGP_OK;
  };
  // the steps of bgp_dense_loo_terms after bgp_dense_compute, member-indexed, with no host check of d in between: a
  // member whose d is not finite and positive runs pass 2 on its own slabs
  auto step = [&](int64_t c0, int mc, const DevProgram*, const DevProgram* dprogs) -> int {
    double* dd = h->d_yerr.p;  // d = diag(K_b^-1), in d_yerr: the build in batch_factor_chunk consumed yerr^2
    BGP_TRY(fill_identity_members(h->d_inv.p, n, mc, s));
    BGP_TRY(potrs_members(h->d_A.p, n, nn, h->d_inv.p, n, n, nn, mc, h->d_tmp.p, s));
    BGP_TRY(slab_diag_members(h->d_inv.p, n, 0, n, dd, mc, nn, n, s));
    if (alpha) BGP_CUDA(cudaMemcpyAsync(alpha + c0 * n, h->d_sol.p, sizeof(double) * mc * n, cudaMemcpyDeviceToHost, s));
    if (d) BGP_CUDA(cudaMemcpyAsync(d + c0 * n, dd, sizeof(double) * mc * n, cudaMemcpyDeviceToHost, s));
    if (!grad) return BGP_OK;
    // pass 2: q and c; beta_b = K_b^-1 q_b (the one-column solve, as for alpha); G_b = diag(sqrt(c_b)) K_b^-1 in place;
    // A_b = -(G_b^T G_b) (lower, mirrored) on the tensor pipe plus 1/2 (beta_b alpha_b^T + alpha_b beta_b^T); then the
    // contraction with A_b given whole, its diagonal into d_diag (whose yerr^2 the build consumed)
    BGP_TRY(loo_weights_members(h->d_sol.p, dd, n, h->d_beta.p, h->d_cw.p, mc, s));
    BGP_TRY(potrs_small_members(h->d_A.p, n, h->d_beta.p, 1, n, h->d_tmp.p, mc, nn, n, s));
    BGP_TRY(scale_rows_members(h->d_inv.p, n, n, n, h->d_cw.p, true, mc, nn, n, s));
    BGP_CUDA(cudaMemsetAsync(h->d_loo_a.p, 0, sizeof(double) * mc * nn, s));
    BGP_TRY(predict_gemm_sub_members(h->d_inv.p, n, h->d_inv.p, n, n, n, n, true, h->d_loo_a.p, n, mc, nn, nn,
                                     h->d_slices, h->d_pdesc, s));
    BGP_TRY(loo_form_a_members(h->d_loo_a.p, n, h->d_sol.p, h->d_beta.p, mc, s));
    BGP_TRY(kmat_grad_contract_members(dprogs, (int)P, h->d_which.p, h->d_x.p, n, h->d_loo_a.p, n, nn, nullptr, 0,
                                       0.0, 1.0, h->d_g.p, P, diag ? h->d_diag.p : nullptr, n, mc, h->d_gp, s));
    if (beta) BGP_CUDA(cudaMemcpyAsync(beta + c0 * n, h->d_beta.p, sizeof(double) * mc * n, cudaMemcpyDeviceToHost, s));
    if (g && P > 0) BGP_CUDA(cudaMemcpyAsync(g + c0 * P, h->d_g.p, sizeof(double) * mc * P, cudaMemcpyDeviceToHost, s));
    if (diag) BGP_CUDA(cudaMemcpyAsync(diag + c0 * n, h->d_diag.p, sizeof(double) * mc * n, cudaMemcpyDeviceToHost, s));
    return BGP_OK;
  };
  // one launch per step for the chunk: the split-K product takes one descriptor per member and slice
  return batch_run(h, bp, x, n, ndim, yerr, r, per_member, 65535 / gsplit, tmp_cols, bufs, setup, step, info,
                   {{alpha, n}, {d, n}, {beta, grad ? n : 0}, {g, grad ? P : 0}, {diag, grad ? n : 0}});
}

int bgp_dense_batch_fisher_terms(bgp_dense_batch_t* h, const bgp_kernel_spec_t* spec, const double* params, int64_t B,
                                 int64_t P, const double* x, int64_t n, int32_t ndim, const double* yerr,
                                 const double* r, const uint32_t* which, const double* v, int32_t nv, const double* dmu,
                                 int32_t nm, double* alpha, double* g, double* diag, double* rows, double* rdiag,
                                 double* kdmu, int32_t* info) {
  if (P > 64) { set_error("gradient supports at most 64 hyper-parameters"); return BGP_ERR_INVALID; }
  if (P > 0 && !which) { set_error("fisher_terms: which is required for a kernel with parameters"); return BGP_ERR_INVALID; }
  if (nv < 0 || (nv > 0 && !v)) { set_error("fisher_terms: invalid white-noise vectors"); return BGP_ERR_INVALID; }
  if (nm < 0 || (nm > 0 && !dmu)) { set_error("fisher_terms: invalid mean gradients"); return BGP_ERR_INVALID; }
  BatchPrograms bp;
  BGP_TRY(batch_begin(h, spec, params, B, P, x, n, ndim, &bp));
  if (B == 0) return BGP_OK;
  cudaStream_t s = h->s;
  const int64_t nn = n * n;
  std::vector<int> krow;  // the kernel rows, then nv white-noise rows, as bgp_dense_fisher_terms orders them
  for (int64_t q = 0; q < P; ++q)
    if (which[q]) krow.push_back((int)q);
  const int64_t nk = (int64_t)krow.size(), nrow = nk + nv;
  // the few-column solve's scratch: K^-1 when n <= 8 (as bgp_dense_fisher_terms sends it), dmu when nm <= 8
  const int64_t tmp_cols = std::max<int64_t>(n <= DS_MAX_RHS ? n : 1, nm <= DS_MAX_RHS ? nm : 1);
  const int64_t nt = (n + 31) / 32;  // the contraction's 32 x 32 tiles
  // the products' split-K plan, bgp_dense_fisher_terms' (no slice buffer with one slice)
  int64_t gsplit = 1, gklen = 0;
  if (nrow) predict_gemm_plan(n, n, n, &gsplit, &gklen);
  const int64_t slices = gsplit > 1 ? gsplit * nn : 0;
  const int64_t planes = nrow ? nn : 0;
  // doubles per member (see include/bgp.h): factor, K^-1, P, T, the split-K slices, the vectors of
  // batch_reserve_common, partials, g, the rows and their diagonals, v and dmu
  const int64_t per_member = 2 * nn + 2 * planes + slices + (4 + tmp_cols) * n + nt * nt * P + P + nrow * (P + n) +
                             (int64_t)(nv + nm) * n;
  const std::vector<ChunkBuf> bufs = {{&h->d_A, nn}, {&h->d_inv, nn}, {&h->d_fp, planes}, {&h->d_ft, planes},
                                      {&h->d_slices, slices}, {&h->d_gp, nt * nt * P}, {&h->d_g, P},
                                      {&h->d_frows, nrow * P}, {&h->d_frd, nrow * n}, {&h->d_fv, (int64_t)nv * n},
                                      {&h->d_fdmu, (int64_t)nm * n}};
  auto setup = [&](int64_t) -> int {
    BGP_TRY(h->d_which.reserve((size_t)std::max<int64_t>(1, P), s));
    if (P > 0) BGP_CUDA(cudaMemcpyAsync(h->d_which.p, which, sizeof(unsigned) * P, cudaMemcpyHostToDevice, s));
    return BGP_OK;
  };
  // the steps of bgp_dense_fisher_terms after bgp_dense_compute, member-indexed, each row one set of launches for the
  // whole chunk; then the mean block's solve, the nm-column bgp_dense_apply_inverse
  auto step = [&](int64_t c0, int mc, const DevProgram*, const DevProgram* dprogs) -> int {
    BGP_TRY(fill_identity_members(h->d_inv.p, n, mc, s));
    BGP_TRY(potrs_members(h->d_A.p, n, nn, h->d_inv.p, n, n, nn, mc, h->d_tmp.p, s));
    if (r) {  // bgp_dense_batch_grad_terms' contraction; the diagonal goes to d_diag, whose yerr^2 the build consumed
      BGP_TRY(kmat_grad_contract_members(dprogs, (int)P, h->d_which.p, h->d_x.p, n, h->d_inv.p, n, nn, h->d_sol.p, n,
                                         1.0, -1.0, h->d_g.p, P, diag ? h->d_diag.p : nullptr, n, mc, h->d_gp, s));
      if (alpha) BGP_CUDA(cudaMemcpyAsync(alpha + c0 * n, h->d_sol.p, sizeof(double) * mc * n, cudaMemcpyDeviceToHost, s));
      if (diag) BGP_CUDA(cudaMemcpyAsync(diag + c0 * n, h->d_diag.p, sizeof(double) * mc * n, cudaMemcpyDeviceToHost, s));
      if (g && P > 0) BGP_CUDA(cudaMemcpyAsync(g + c0 * P, h->d_g.p, sizeof(double) * mc * P, cudaMemcpyDeviceToHost, s));
    }
    if (nv)
      BGP_CUDA(cudaMemcpyAsync(h->d_fv.p, v + c0 * nv * n, sizeof(double) * mc * nv * n, cudaMemcpyHostToDevice, s));
    const size_t bytes = sizeof(double) * (size_t)mc * (size_t)nn;
    for (int64_t row = 0; row < nrow; ++row) {
      double cm = 1.0;
      if (row < nk) {
        BGP_TRY(kmat_gradient_plane_members(dprogs, (int)P, krow[(size_t)row], h->d_x.p, n, h->d_fp.p, n, nn, mc, s));
        BGP_CUDA(cudaMemsetAsync(h->d_ft.p, 0, bytes, s));
        BGP_TRY(predict_gemm_sub_members(h->d_inv.p, n, h->d_fp.p, n, n, n, n, false, h->d_ft.p, n, mc, nn, nn,
                                         h->d_slices, h->d_pdesc, s));
        BGP_CUDA(cudaMemsetAsync(h->d_fp.p, 0, bytes, s));
        BGP_TRY(predict_gemm_sub_bt_members(h->d_inv.p, n, h->d_ft.p, n, n, n, n, true, h->d_fp.p, n, mc, nn, nn,
                                            h->d_slices, h->d_pdesc, s));
      } else {
        BGP_CUDA(cudaMemcpyAsync(h->d_ft.p, h->d_inv.p, bytes, cudaMemcpyDeviceToDevice, s));
        BGP_TRY(scale_rows_members(h->d_ft.p, n, n, n, h->d_fv.p + (row - nk) * n, false, mc, nn, (int64_t)nv * n, s));
        BGP_CUDA(cudaMemsetAsync(h->d_fp.p, 0, bytes, s));
        BGP_TRY(predict_gemm_sub_members(h->d_inv.p, n, h->d_ft.p, n, n, n, n, true, h->d_fp.p, n, mc, nn, nn,
                                         h->d_slices, h->d_pdesc, s));
        cm = -1.0;
      }
      BGP_TRY(kmat_grad_contract_members(dprogs, (int)P, h->d_which.p, h->d_x.p, n, h->d_fp.p, n, nn, nullptr, 0, 0.0,
                                         cm, h->d_frows.p + row * P, nrow * P, h->d_frd.p + row * n, nrow * n, mc,
                                         h->d_gp, s));
    }
    if (rows && nrow * P > 0)
      BGP_CUDA(cudaMemcpyAsync(rows + c0 * nrow * P, h->d_frows.p, sizeof(double) * mc * nrow * P,
                               cudaMemcpyDeviceToHost, s));
    if (rdiag && nrow > 0)
      BGP_CUDA(cudaMemcpyAsync(rdiag + c0 * nrow * n, h->d_frd.p, sizeof(double) * mc * nrow * n,
                               cudaMemcpyDeviceToHost, s));
    if (nm) {
      const int64_t len = (int64_t)nm * n;
      BGP_CUDA(cudaMemcpyAsync(h->d_fdmu.p, dmu + c0 * len, sizeof(double) * mc * len, cudaMemcpyHostToDevice, s));
      BGP_TRY(potrs_members(h->d_A.p, n, nn, h->d_fdmu.p, nm, n, len, mc, h->d_tmp.p, s));
      if (kdmu) BGP_CUDA(cudaMemcpyAsync(kdmu + c0 * len, h->d_fdmu.p, sizeof(double) * mc * len, cudaMemcpyDeviceToHost, s));
    }
    return BGP_OK;
  };
  // one launch per step for the chunk: the split-K products take one descriptor per member and slice
  const int64_t rl = r ? 1 : 0;
  return batch_run(h, bp, x, n, ndim, yerr, r, per_member, 65535 / gsplit, tmp_cols, bufs, setup, step, info,
                   {{alpha, rl * n}, {g, rl * P}, {diag, rl * n}, {rows, nrow * P}, {rdiag, nrow * n},
                    {kdmu, (int64_t)nm * n}});
}

int bgp_dense_batch_predict(bgp_dense_batch_t* h, const bgp_kernel_spec_t* spec, const double* params, int64_t B,
                            int64_t P, const double* x, int64_t n, int32_t ndim, const double* yerr, const double* r,
                            const double* xs, int64_t ns, int32_t what, double* mean, double* out, int32_t* info) {
  if (out && what != BGP_PREDICT_VAR && what != BGP_PREDICT_COV) { set_error("invalid prediction kind %d", what); return BGP_ERR_INVALID; }
  if (ns < 0) { set_error("negative number of test points"); return BGP_ERR_INVALID; }
  BatchPrograms bp;
  BGP_TRY(batch_begin(h, spec, params, B, P, x, n, ndim, &bp));
  if (B == 0) return BGP_OK;
  cudaStream_t s = h->s;
  const bool var = out && what == BGP_PREDICT_VAR, cov = out && what == BGP_PREDICT_COV;
  const int64_t nn = n * n;
  const BatchTestPlan tp(n, ns, var, cov);
  const int64_t tmp_cols = (var || cov) ? DS_MAX_RHS : 1;
  // doubles per member (see include/bgp.h)
  int64_t per_member = nn + (4 + tmp_cols) * n + ns + tp.mvp;
  if (var) per_member += n * tp.c + 2 * tp.c + tp.vp;
  if (cov) per_member += n * ns + ns * ns * (1 + tp.gsplit);
  std::vector<ChunkBuf> bufs = {{&h->d_A, nn}, {&h->d_tmp, n * tmp_cols}, {&h->d_mean, ns}, {&h->d_mvp, tp.mvp}};
  if (var) bufs.insert(bufs.end(), {{&h->d_W, n * tp.c}, {&h->d_kd, tp.c}, {&h->d_var, tp.c}, {&h->d_vp, tp.vp}});
  if (cov) bufs.insert(bufs.end(), {{&h->d_W, n * ns}, {&h->d_C, ns * ns}, {&h->d_slices, ns * ns * tp.gsplit}});
  auto step = [&](int64_t c0, int mc, const DevProgram* progs, const DevProgram* dprogs) -> int {
    BGP_TRY(batch_mean_chunk(h, dprogs, ndim, mc, n, ns));
    if (ns > 0)
      BGP_CUDA(cudaMemcpyAsync(mean + c0 * ns, h->d_mean.p, sizeof(double) * mc * ns, cudaMemcpyDeviceToHost, s));
    if (var) {
      for (int64_t j0 = 0; j0 < ns; j0 += tp.c)
        BGP_TRY(batch_var_chunk(h, progs, dprogs, mc, n, ndim, tp.c, j0, std::min(tp.c, ns - j0), out + c0 * ns, ns));
    } else if (cov && ns > 0) {
      BGP_TRY(batch_cov_chunk(h, progs, dprogs, mc, n, ndim, ns, tp.c));
      BGP_CUDA(cudaMemcpyAsync(out + c0 * ns * ns, h->d_C.p, sizeof(double) * mc * ns * ns, cudaMemcpyDeviceToHost, s));
    }
    return BGP_OK;
  };
  // COV: one DMMA launch per chunk, one descriptor per member and split-K slice
  return batch_run(h, bp, x, n, ndim, yerr, r, per_member, 65535 / tp.gsplit, tmp_cols, bufs,
                   [&](int64_t) { return batch_upload_xs(h, xs, ns, ndim); }, step, info,
                   {{mean, ns}, {out, var ? ns : cov ? ns * ns : 0}});
}

int bgp_dense_batch_predict_grad(bgp_dense_batch_t* h, const bgp_kernel_spec_t* spec, const double* params, int64_t B,
                                 int64_t P, const double* x, int64_t n, int32_t ndim, const double* yerr,
                                 const double* r, const double* xs, int64_t ns, int32_t with_var, double* mean,
                                 double* dmu, double* var, double* dvar, int32_t* info) {
  if (ndim > BGP_MAX_DIM) { set_error("input-coordinate gradients support at most %d dimensions (got %d)", BGP_MAX_DIM, ndim); return BGP_ERR_INVALID; }
  if (ns < 0) { set_error("negative number of test points"); return BGP_ERR_INVALID; }
  if (with_var && (!var || !dvar)) { set_error("with_var needs the var and dvar outputs"); return BGP_ERR_INVALID; }
  BatchPrograms bp;
  BGP_TRY(batch_begin(h, spec, params, B, P, x, n, ndim, &bp));
  if (B == 0) return BGP_OK;
  cudaStream_t s = h->s;
  const int64_t nn = n * n;
  const int64_t nd = ndim;
  // bgp_dense_batch_predict's mean and VAR workspace, plus dmu, a chunk of dvar and the contraction partials (the
  // larger of dmu's and a dvar chunk's: they run one after the other)
  const BatchTestPlan tp(n, ns, with_var, false);
  const int64_t c = tp.c;
  int64_t xgp = x1_grad_partial_size(ns, n, ndim);
  if (with_var) xgp = std::max(xgp, std::max(x1_grad_partial_size(c, n, ndim), x1_grad_partial_size(tp.tail, n, ndim)));
  const int64_t tmp_cols = with_var ? DS_MAX_RHS : 1;
  // doubles per member (see include/bgp.h)
  int64_t per_member = nn + (4 + tmp_cols) * n + ns + tp.mvp + ns * nd + xgp;
  if (with_var) per_member += n * c + 2 * c + tp.vp + c * nd;
  std::vector<ChunkBuf> bufs = {{&h->d_A, nn},       {&h->d_tmp, n * tmp_cols}, {&h->d_mean, ns},
                                {&h->d_mvp, tp.mvp}, {&h->d_dmu, ns * nd},      {&h->d_xgp, xgp}};
  if (with_var)
    bufs.insert(bufs.end(), {{&h->d_W, n * c}, {&h->d_kd, c}, {&h->d_var, c}, {&h->d_vp, tp.vp}, {&h->d_dvar, c * nd}});
  // the steps of bgp_dense_batch_predict (factor, alpha, mean, VAR), then those of bgp_dense_predict_grad, with a
  // member index.  A member whose K is not positive definite runs the later steps on its own slabs.
  auto step = [&](int64_t c0, int mc, const DevProgram* progs, const DevProgram* dprogs) -> int {
    if (ns > 0) {
      BGP_TRY(batch_mean_chunk(h, dprogs, ndim, mc, n, ns));
      BGP_CUDA(cudaMemcpyAsync(mean + c0 * ns, h->d_mean.p, sizeof(double) * mc * ns, cudaMemcpyDeviceToHost, s));
      // dmu_b = sum_j d1 k_b(x*, x_j) alpha_bj: GP.grad_predict's kernel.x1_gradient_matvec(xs, x, alpha)
      BGP_TRY(kmat_x1_grad_matvec_members(progs, dprogs, mc, h->d_xs.p, ns, h->d_x.p, n, h->d_sol.p, 0, n, 1.0, 0,
                                          h->d_dmu.p, ns * nd, h->d_xgp, s));
      BGP_CUDA(cudaMemcpyAsync(dmu + c0 * ns * nd, h->d_dmu.p, sizeof(double) * mc * ns * nd, cudaMemcpyDeviceToHost, s));
    }
    if (!with_var) return BGP_OK;
    const int64_t ldw = (int64_t)mc * n;
    for (int64_t j0 = 0; j0 < ns; j0 += c) {
      const int64_t nc = std::min(c, ns - j0);
      BGP_TRY(batch_var_chunk(h, progs, dprogs, mc, n, ndim, c, j0, nc, var + c0 * ns, ns));
      // bgp_dense_predict_grad's: W <- L_b^-T W = K_b^-1 K_b(x, x*), dvar = dprior - 2 sum_j d1 k_b(x*, x_j) W_j
      BGP_TRY(trsm_bwd_members(h->d_A.p, n, nn, h->d_W.p, nc, ldw, n, mc, h->d_tmp.p, ldw, s));
      BGP_TRY(kmat_x1_grad_matvec_members(progs, dprogs, mc, h->d_xs.p + j0 * nd, nc, h->d_x.p, n, h->d_W.p, ldw, n,
                                          -2.0, 1, h->d_dvar.p, c * nd, h->d_xgp, s));
      BGP_CUDA(cudaMemcpy2DAsync(dvar + (c0 * ns + j0) * nd, sizeof(double) * ns * nd, h->d_dvar.p,
                                 sizeof(double) * c * nd, sizeof(double) * nc * nd, mc, cudaMemcpyDeviceToHost, s));
    }
    return BGP_OK;
  };
  return batch_run(h, bp, x, n, ndim, yerr, r, per_member, 65535, tmp_cols, bufs,
                   [&](int64_t) { return batch_upload_xs(h, xs, ns, ndim); }, step, info,
                   {{mean, ns}, {var, with_var ? ns : 0}, {dmu, ns * nd}, {dvar, with_var ? ns * nd : 0}});
}

int bgp_dense_batch_sample(bgp_dense_batch_t* h, const bgp_kernel_spec_t* spec, const double* params, int64_t B,
                           int64_t P, const double* x, int64_t n, int32_t ndim, const double* yerr, const double* r,
                           const double* xs, int64_t ns, const double* mean_add, const double* z, int64_t size,
                           double jitter, double* draws, int32_t* info, int32_t* draw_info) {
  BGP_TRY(mvn_sample_check(ns, size, jitter));
  BatchPrograms bp;
  BGP_TRY(batch_begin(h, spec, params, B, P, x, n, ndim, &bp));
  if (B == 0) return BGP_OK;
  cudaStream_t s = h->s;
  const bool draw = ns > 0 && size > 0;
  const int64_t nn = n * n;
  const int64_t dsize = size * ns;  // a member's draws
  // bgp_dense_batch_predict's COV workspace plus z, the draws and the mean
  const BatchTestPlan tp(n, ns, false, draw);
  const int64_t tmp_cols = DS_MAX_RHS;
  const int64_t per_member =
      nn + (4 + tmp_cols) * n + ns + tp.mvp + n * ns + ns * ns * (1 + tp.gsplit) + 2 * dsize + ns;
  // one launch per step for the chunk: the split-K product and the draws' DMMA product each take one descriptor per
  // member and slice, at most 65535 per launch
  int64_t cap = 65535 / tp.gsplit;
  if (draw && mvn_product_descs(ns, size) > 0) cap = std::min<int64_t>(cap, 65535 / mvn_product_descs(ns, size));
  std::vector<ChunkBuf> bufs = {{&h->d_A, nn}, {&h->d_tmp, n * tmp_cols}, {&h->d_mean, ns}, {&h->d_mvp, tp.mvp}};
  if (draw)
    bufs.insert(bufs.end(), {{&h->d_W, n * ns}, {&h->d_C, ns * ns}, {&h->d_slices, ns * ns * tp.gsplit},
                             {&h->d_madd, ns}, {&h->d_z, dsize}, {&h->d_draws, dsize}});
  auto setup = [&](int64_t c) -> int {
    BGP_TRY(h->d_dinfo.reserve((size_t)c, s));
    return batch_upload_xs(h, xs, ns, ndim);
  };
  // the steps of bgp_dense_batch_predict (factor, alpha, mean, COV), then those of bgp_dense_sample's draw with a
  // member index.  A member whose K is not positive definite runs every later step on its own slabs, which no other
  // member reads; nothing synchronises inside the chunk.
  auto step = [&](int64_t c0, int mc, const DevProgram* progs, const DevProgram* dprogs) -> int {
    if (!draw) {
      for (int m = 0; m < mc; ++m) draw_info[c0 + m] = 0;
      return BGP_OK;
    }
    BGP_TRY(batch_mean_chunk(h, dprogs, ndim, mc, n, ns));
    BGP_CUDA(cudaMemcpyAsync(h->d_madd.p, mean_add + c0 * ns, sizeof(double) * mc * ns, cudaMemcpyHostToDevice, s));
    BGP_CUDA(cudaMemcpyAsync(h->d_z.p, z + c0 * dsize, sizeof(double) * mc * dsize, cudaMemcpyHostToDevice, s));
    add_into_kernel<<<(unsigned)std::min<int64_t>((mc * ns + 255) / 256, 1184), 256, 0, s>>>(h->d_mean.p, h->d_madd.p,
                                                                                            mc * ns);
    BGP_LAUNCH_CHECK();
    BGP_TRY(batch_cov_chunk(h, progs, dprogs, mc, n, ndim, ns, tp.c));
    BGP_TRY(mvn_factor_members(h->d_C.p, ns, jitter, mc, h->d_dinfo.p, nullptr, h->d_gdesc, s));
    BGP_TRY(mvn_product_members(h->d_C.p, ns, h->d_madd.p, ns, h->d_z.p, size, h->d_draws.p, mc, h->d_sdesc, s));
    BGP_CUDA(cudaMemcpyAsync(draws + c0 * dsize, h->d_draws.p, sizeof(double) * mc * dsize, cudaMemcpyDeviceToHost, s));
    BGP_CUDA(cudaMemcpyAsync(draw_info + c0, h->d_dinfo.p, sizeof(int) * mc, cudaMemcpyDeviceToHost, s));
    return BGP_OK;
  };
  BGP_TRY(batch_run(h, bp, x, n, ndim, yerr, r, per_member, cap, tmp_cols, bufs, setup, step, info, {{draws, dsize}}));
  // a failed member has no draw_info; a failed draw's rows are NaN as well
  for (int64_t b = 0; b < B; ++b) {
    if (info[b] != 0)
      draw_info[b] = 0;
    else if (draw_info[b] != 0)
      std::fill(draws + b * dsize, draws + (b + 1) * dsize, std::nan(""));
  }
  return BGP_OK;
}

}  // extern "C"
