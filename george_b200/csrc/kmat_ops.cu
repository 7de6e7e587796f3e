// kmat_ops.cu — matrix-free consumers of the covariance function: nothing here ever materialises a kernel matrix.
//
//   kmat_matvec_kernel       out = K(x1, x2) V   (+ diag . V)      -> GP.predict's mean  K(x*, x) alpha
//                            (reference: kernel.get_value(xs, x) then numpy dot, src/george/gp.py:524-528 over
//                             kernel_interface.cpp:47-60), and the full-size round-trip check  K (K^-1 y) == y.
//   kmat_grad_contract_kernel  g_p = sum_ij A_ij dK_ij/dtheta_p     -> GP.grad_log_likelihood's kernel term
//                            (reference: kernel.get_gradient(x) -> (n, n, P) tensor, then
//                             0.5 * einsum("ijk,ij", dK, alpha alpha^T - K^-1), src/george/gp.py:437-466 over
//                             kernel_interface.cpp:109-125).  A is read once (8 n^2 bytes); the (n, n, P) tensor is never
//                             formed.
//   predict_var_* / predict_gemm_sub  GP.predict's variance and covariance from K(x, x*) and K^-1 K(x, x*) chunks
//                            that the solvers stream (dense.cu, hodlr.cu; reference gp.py:534-545).
//   kmat_x1_grad_matvec_kernel  out_i = sum_j dk(x1_i, x2_j)/dx1_i V_ji  -> GP.grad_predict's dmu (V = alpha, shared)
//                            and dvar (V = K^-1 K(x, x*), one column per test point); the (n1, n2, ndim) gradient
//                            tensor is never formed.
//
// Roofline: matvec is FP64-ALU bound (one covariance evaluation per (i, j), no HBM traffic beyond x and V);
// the contraction reads A once -> HBM bound at 8 B per pair for cheap kernels, FP64 bound for the gradient of
// expensive ones.  Partial sums are written per CTA and reduced by a second tiny kernel in a fixed order, so results
// are run-to-run deterministic (no atomics).
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <vector>

#include "common.cuh"
#include "gemm_dmma.cuh"
#include "kernel_eval.cuh"

namespace bgp {
int upload_program(const DevProgram& P, DevBuf<DevProgram>& buf, cudaStream_t s);

constexpr int MV_TI = 64;        // rows per CTA
constexpr int MV_TJ = 512;       // columns staged per iteration
constexpr int MV_THREADS = 256;  // 64 rows x 4 column lanes
constexpr int MV_NR = 4;         // right-hand sides per launch

struct MvSmem {
  DevProgram prog;
  uint64_t bar;
};

// partial[(split * n1 + i) * MV_NR + c] = sum_{j in split's chunks} k(x1_i, x2_j) V[j + c*ldv]
template <typename Fn>
__device__ __forceinline__ void matvec_tile(const Fn& fn, int nd, const double* sx1, const double* sx2,
                                            const double* sv, int ni, int nj, int row, int lane4, double (&acc)[MV_NR]) {
  if (row >= ni) return;
  const double* xi = sx1 + row * nd;
  for (int j = lane4; j < nj; j += MV_THREADS / MV_TI) {
    const double k = fn(xi, sx2 + j * nd);
#pragma unroll
    for (int c = 0; c < MV_NR; ++c) acc[c] = fma(k, sv[c * MV_TJ + j], acc[c]);
  }
}

// STAGED: the coordinates are staged in shared memory; otherwise (inputs too wide for the cap, tile_kernel_for) they
// are read from global memory, with the same evaluation order
template <bool STAGED>
__global__ void __launch_bounds__(MV_THREADS) kmat_matvec_kernel(const DevProgram* __restrict__ gprog,
                                                                 const double* __restrict__ x1, int64_t n1,
                                                                 const double* __restrict__ x2, int64_t n2,
                                                                 const double* __restrict__ V, int64_t ldv, int nrhs,
                                                                 double* __restrict__ partial, int chunks_per_split,
                                                                 int64_t vstride, int64_t pstride) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  MvSmem* S = reinterpret_cast<MvSmem*>(smem_raw);
  gprog += blockIdx.z;  // member blockIdx.z of a batch: its program, V + z * vstride, partial + z * pstride
  V += blockIdx.z * vstride;
  partial += blockIdx.z * pstride;
  const int nd = gprog->ndim;
  const int snd = STAGED ? nd : 0;  // doubles per staged point
  double* sx1 = reinterpret_cast<double*>(smem_raw + ((sizeof(MvSmem) + 15) & ~size_t(15)));
  double* sx2 = sx1 + MV_TI * snd + ((MV_TI * snd) & 1);
  double* sv = sx2 + MV_TJ * snd;          // MV_NR x MV_TJ
  double* red = sv + MV_NR * MV_TJ;         // MV_THREADS x MV_NR

  stage_program(&S->prog, gprog);
  if (STAGED && threadIdx.x == 0) { mbar_init(&S->bar, 1); mbar_fence_init(); }
  __syncthreads();
  uint32_t phase = 0;

  const int64_t i0 = (int64_t)blockIdx.x * MV_TI;
  const int ni = (int)min((int64_t)MV_TI, n1 - i0);
  const double* X1 = x1 + i0 * nd;
  if (STAGED) {
    load_coords(sx1, X1, ni * nd, &S->bar, phase);
    X1 = sx1;
  }

  const int row = threadIdx.x & (MV_TI - 1), lane4 = threadIdx.x / MV_TI;
  double acc[MV_NR];
#pragma unroll
  for (int c = 0; c < MV_NR; ++c) acc[c] = 0.0;

  const int64_t nchunks = (n2 + MV_TJ - 1) / MV_TJ;
  const int64_t c_begin = (int64_t)blockIdx.y * chunks_per_split;
  const int64_t c_end = min(nchunks, c_begin + chunks_per_split);
  for (int64_t ch = c_begin; ch < c_end; ++ch) {
    const int64_t j0 = ch * MV_TJ;
    const int nj = (int)min((int64_t)MV_TJ, n2 - j0);
    __syncthreads();  // previous iteration's readers are done with sx2 / sv
    const double* X2 = x2 + j0 * nd;
    if (STAGED) {
      load_coords(sx2, X2, nj * nd, &S->bar, phase);
      X2 = sx2;
    }
    for (int t = threadIdx.x; t < MV_NR * MV_TJ; t += MV_THREADS) {
      const int c = t / MV_TJ, j = t - c * MV_TJ;
      sv[t] = (c < nrhs && j < nj) ? V[(int64_t)c * ldv + j0 + j] : 0.0;
    }
    __syncthreads();
    BGP_DISPATCH_SHAPE(S->prog, matvec_tile(fn, nd, X1, X2, sv, ni, nj, row, lane4, acc));
  }
  // combine the 4 column lanes of each row (fixed order), one partial per (split, row, rhs)
#pragma unroll
  for (int c = 0; c < MV_NR; ++c) red[threadIdx.x * MV_NR + c] = acc[c];
  __syncthreads();
  if (lane4 == 0 && row < ni) {
#pragma unroll
    for (int c = 0; c < MV_NR; ++c) {
      double s = red[row * MV_NR + c];
      for (int q = 1; q < MV_THREADS / MV_TI; ++q) s += red[(q * MV_TI + row) * MV_NR + c];
      partial[((int64_t)blockIdx.y * n1 + i0 + row) * MV_NR + c] = s;
    }
  }
}

// out[i + c*ldo] = sum_s partial[(s*n1 + i)*MV_NR + c]  (+ diag[i] * V[i + c*ldv])
// (member blockIdx.y of a batch: partial + y * pstride, V + y * vstride, out + y * ostride)
__global__ void kmat_matvec_reduce_kernel(const double* __restrict__ partial, int64_t n1, int nsplit, int nrhs,
                                          const double* __restrict__ diag, const double* __restrict__ V, int64_t ldv,
                                          double* __restrict__ out, int64_t ldo, int64_t pstride, int64_t vstride,
                                          int64_t ostride) {
  partial += blockIdx.y * pstride;
  V += blockIdx.y * vstride;
  out += blockIdx.y * ostride;
  const int64_t total = n1 * nrhs;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t c = t / n1, i = t - c * n1;
    double s = 0.0;
    for (int sp = 0; sp < nsplit; ++sp) s += partial[((int64_t)sp * n1 + i) * MV_NR + c];
    if (diag) s = fma(diag[i], V[c * ldv + i], s);
    out[c * ldo + i] = s;
  }
}

// dynamic shared memory of the matvec staging the coordinates of nd-dimensional points (nd = 0: none); the cap is the
// most the staged matvec may take
constexpr size_t MV_SMEM_CAP = 160 * 1024;
static size_t matvec_smem(int nd) {
  return ((sizeof(MvSmem) + 15) & ~size_t(15)) +
         sizeof(double) * ((size_t)MV_TI * nd + 1 + (size_t)MV_TJ * nd + (size_t)MV_NR * MV_TJ + (size_t)MV_THREADS * MV_NR);
}

// The column split of K(x1, x2) V (n1 x n2): nsplit groups of cps 512-column chunks, one partial per (split, row).
// Enough CTAs for ~8 per SM; when there are few row tiles (predict at a handful of points) split the columns instead.
int matvec_plan(int64_t n1, int64_t n2, int64_t* nsplit_out, int* cps_out) {
  const int64_t row_tiles = (n1 + MV_TI - 1) / MV_TI;
  const int64_t nchunks = (n2 + MV_TJ - 1) / MV_TJ;
  int64_t nsplit = std::max<int64_t>(1, std::min<int64_t>(nchunks, (8 * (int64_t)num_sms() + row_tiles - 1) / row_tiles));
  const int cps = (int)((nchunks + nsplit - 1) / nsplit);
  nsplit = (nchunks + cps - 1) / cps;
  if (row_tiles > 0x7fffffffLL || nsplit > 65535) { set_error("kmat_matvec: problem too large for one launch"); return BGP_ERR_INVALID; }
  *nsplit_out = nsplit;
  *cps_out = cps;
  return BGP_OK;
}
// doubles of matvec partials per member (one right-hand side group)
int64_t matvec_partial_size(int64_t n1, int64_t n2) {
  int64_t nsplit = 1;
  int cps = 1;
  if (n1 <= 0 || n2 <= 0 || matvec_plan(n1, n2, &nsplit, &cps) != BGP_OK) return 0;
  return nsplit * n1 * MV_NR;
}

// out (n1 x nrhs, column-major ldo) = K(x1, x2) V (n2 x nrhs, column-major ldv) [+ diag .* V, only when n1 == n2]
int kmat_matvec_launch(const DevProgram* dprog, int nd, const double* x1, int64_t n1, const double* x2, int64_t n2,
                       const double* diag, const double* V, int64_t ldv, int64_t nrhs, double* out, int64_t ldo,
                       DevBuf<double>& scratch, cudaStream_t s) {
  if (n1 <= 0 || nrhs <= 0) return BGP_OK;
  if (n2 <= 0) {
    for (int64_t c = 0; c < nrhs; ++c) BGP_CUDA(cudaMemsetAsync(out + c * ldo, 0, sizeof(double) * n1, s));
    return BGP_OK;
  }
  size_t smem;
  const auto kern = tile_kernel_for(kmat_matvec_kernel<true>, kmat_matvec_kernel<false>, matvec_smem(nd), matvec_smem(0),
                                    MV_SMEM_CAP, &smem);
  const int64_t row_tiles = (n1 + MV_TI - 1) / MV_TI;
  int64_t nsplit;
  int cps;
  BGP_TRY(matvec_plan(n1, n2, &nsplit, &cps));
  BGP_TRY(scratch.reserve((size_t)nsplit * (size_t)n1 * MV_NR, s));
  for (int64_t c0 = 0; c0 < nrhs; c0 += MV_NR) {
    const int nc = (int)std::min<int64_t>(MV_NR, nrhs - c0);
    dim3 grid((unsigned)row_tiles, (unsigned)nsplit);
    kern<<<grid, MV_THREADS, smem, s>>>(dprog, x1, n1, x2, n2, V + c0 * ldv, ldv, nc, scratch.p, cps, 0, 0);
    BGP_LAUNCH_CHECK();
    const int blocks = (int)std::min<int64_t>((n1 * nc + 255) / 256, 8 * (int64_t)num_sms());
    kmat_matvec_reduce_kernel<<<blocks, 256, 0, s>>>(scratch.p, n1, (int)nsplit, nc, diag, V + c0 * ldv, ldv,
                                                     out + c0 * ldo, ldo, 0, 0, 0);
    BGP_LAUNCH_CHECK();
  }
  return BGP_OK;
}

// `members` products of one right-hand side on the same x1, x2 in one launch each: member b computes
// out + b * ostride (n1) = K_b(x1, x2) (V + b * vstride) with program dprogs[b], exactly as kmat_matvec_launch computes
// it for that program (the same split plan, the same per-row order).  partial: members * matvec_partial_size(n1, n2).
int kmat_matvec_batch_launch(const DevProgram* dprogs, int nd, int members, const double* x1, int64_t n1,
                             const double* x2, int64_t n2, const double* V, int64_t vstride, double* out,
                             int64_t ostride, double* partial, cudaStream_t s) {
  if (n1 <= 0 || members <= 0) return BGP_OK;
  if (members > 65535) { set_error("kmat_matvec: more than 65535 members in one launch"); return BGP_ERR_INVALID; }
  if (n2 <= 0) {
    BGP_CUDA(cudaMemset2DAsync(out, sizeof(double) * ostride, 0, sizeof(double) * n1, members, s));
    return BGP_OK;
  }
  const int64_t row_tiles = (n1 + MV_TI - 1) / MV_TI;
  int64_t nsplit;
  int cps;
  BGP_TRY(matvec_plan(n1, n2, &nsplit, &cps));
  const int64_t pstride = nsplit * n1 * MV_NR;
  size_t smem;
  const auto kern = tile_kernel_for(kmat_matvec_kernel<true>, kmat_matvec_kernel<false>, matvec_smem(nd), matvec_smem(0),
                                    MV_SMEM_CAP, &smem);
  kern<<<dim3((unsigned)row_tiles, (unsigned)nsplit, (unsigned)members), MV_THREADS, smem, s>>>(
      dprogs, x1, n1, x2, n2, V, n2, 1, partial, cps, vstride, pstride);
  BGP_LAUNCH_CHECK();
  const int blocks = (int)std::min<int64_t>((n1 + 255) / 256, 8 * (int64_t)num_sms());
  kmat_matvec_reduce_kernel<<<dim3(blocks, members), 256, 0, s>>>(partial, n1, (int)nsplit, 1, nullptr, V, n2, out, n1,
                                                                  pstride, vstride, ostride);
  BGP_LAUNCH_CHECK();
  return BGP_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Input-gradient contraction (GP.grad_predict):
//     out[i*nd + q] = (add_prior ? d k(x1_i, x1_i) / d x1_iq : 0) + scale * sum_j d k(x1_i, x2_j) / d x1_iq * V_ji
// V_ji = V[j] (ldv == 0: one vector shared by every i, the mean's alpha) or V[i*ldv + j] (column i of an n2 x n1
// column-major matrix, the variance's W = K^-1 K(x, x*)).  The prior term d k(x, x)/dx = (d1 + d2) k(x, x) is taken as
// 2 d1 k(x, x), every kernel being symmetric; it is 0 for stationary leaves.
// Tiles of XG_TI test points against staged XG_TJ-point chunks of x2, as the matvec; the chunks are split over
// blockIdx.y when there are few test points.  One warp takes one test point at a time with its lanes along j, so W is
// read coalesced (8 * n2 * n1 bytes in all, the kernel's only large HBM traffic).  Each warp's sum over a chunk goes to
// a per-point accumulator in shared memory owned by that warp; per-CTA partials are summed over the splits in a fixed
// order by x1_grad_reduce_kernel.  No atomics: identical calls give identical bits.
// Member blockIdx.z of a batch (bgp_dense_batch_predict_grad) contracts with its own program gprog[z] and V + z * vstride
// and writes partial + z * pstride; x1 and x2 are shared.  A single contraction launches one member with zero strides.
// ---------------------------------------------------------------------------------------------------------------
constexpr int XG_TI = 32;
constexpr int XG_TJ = 512;
constexpr int XG_THREADS = 256;
constexpr int XG_WARPS = XG_THREADS / 32;

static size_t x1_grad_smem(int nd) {
  return ((sizeof(DevProgram) + 15) & ~size_t(15)) +
         sizeof(double) * ((size_t)XG_TI * nd + (size_t)XG_TJ * nd + XG_TJ + (size_t)XG_TI * nd);
}

// partial[(split * n1 + i) * nd + q] = sum_{j in split's chunks} d k(x1_i, x2_j) / d x1_iq V_ji
template <int SHAPE>
__global__ void __launch_bounds__(XG_THREADS) kmat_x1_grad_matvec_kernel(const DevProgram* __restrict__ gprog,
                                                                         const double* __restrict__ x1, int64_t n1,
                                                                         const double* __restrict__ x2, int64_t n2,
                                                                         const double* __restrict__ V, int64_t ldv,
                                                                         double* __restrict__ partial,
                                                                         int chunks_per_split, int64_t vstride,
                                                                         int64_t pstride) {
  gprog += blockIdx.z;
  V += blockIdx.z * vstride;
  partial += blockIdx.z * pstride;
  using Eval = X1GradEval<SHAPE>;
  constexpr int NDMAX = Eval::type::NDMAX;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  DevProgram* prog = reinterpret_cast<DevProgram*>(smem_raw);
  const int nd = gprog->ndim;
  double* sx1 = reinterpret_cast<double*>(smem_raw + ((sizeof(DevProgram) + 15) & ~size_t(15)));
  double* sx2 = sx1 + XG_TI * nd;
  double* sv = sx2 + XG_TJ * nd;  // the chunk of V (ldv == 0)
  double* sacc = sv + XG_TJ;      // XG_TI x nd: per-point sums, point p owned by warp p % XG_WARPS
  stage_program(prog, gprog);
  const int64_t i0 = (int64_t)blockIdx.x * XG_TI;
  const int ni = (int)min((int64_t)XG_TI, n1 - i0);
  for (int t = threadIdx.x; t < ni * nd; t += XG_THREADS) sx1[t] = x1[i0 * nd + t];
  for (int t = threadIdx.x; t < XG_TI * nd; t += XG_THREADS) sacc[t] = 0.0;
  __syncthreads();
  const typename Eval::type fn = Eval::make(prog);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  const int64_t nchunks = (n2 + XG_TJ - 1) / XG_TJ;
  const int64_t c_begin = (int64_t)blockIdx.y * chunks_per_split;
  const int64_t c_end = min(nchunks, c_begin + chunks_per_split);
  for (int64_t ch = c_begin; ch < c_end; ++ch) {
    const int64_t j0 = ch * XG_TJ;
    const int nj = (int)min((int64_t)XG_TJ, n2 - j0);
    __syncthreads();  // previous iteration's readers are done with sx2 / sv
    for (int t = threadIdx.x; t < nj * nd; t += XG_THREADS) sx2[t] = x2[j0 * nd + t];
    if (ldv == 0)
      for (int t = threadIdx.x; t < nj; t += XG_THREADS) sv[t] = V[j0 + t];
    __syncthreads();
    for (int p = warp; p < ni; p += XG_WARPS) {
      const double* xi = sx1 + p * nd;
      const double* w = V + (i0 + p) * ldv + j0;
      double acc[NDMAX];
#pragma unroll
      for (int q = 0; q < NDMAX; ++q) acc[q] = 0.0;
      for (int j = lane; j < nj; j += 32) {
        const double v = ldv ? w[j] : sv[j];
        double g[NDMAX];
        fn(xi, sx2 + j * nd, g);
#pragma unroll
        for (int q = 0; q < NDMAX; ++q)
          if (q < nd) acc[q] = fma(g[q], v, acc[q]);
      }
#pragma unroll
      for (int q = 0; q < NDMAX; ++q) {
        if (q < nd) {  // uniform across the warp
          const double s = warp_sum(acc[q]);
          if (lane == 0) sacc[p * nd + q] += s;
        }
      }
    }
  }
  __syncthreads();
  for (int t = threadIdx.x; t < ni * nd; t += XG_THREADS) partial[((int64_t)blockIdx.y * n1 + i0) * nd + t] = sacc[t];
}

// out[i*nd + q] = (add_prior ? 2 d1 k(x1_i, x1_i)_q : 0) + scale * sum_s partial[(s*n1 + i)*nd + q], s ascending
// (member blockIdx.y: the prior term of gprog[y], partial + y * pstride, out + y * ostride)
__global__ void x1_grad_reduce_kernel(const DevProgram* __restrict__ gprog, const double* __restrict__ x1, int64_t n1,
                                      const double* __restrict__ partial, int64_t nsplit, double scale, int add_prior,
                                      double* __restrict__ out, int64_t pstride, int64_t ostride) {
  gprog += blockIdx.y;
  partial += blockIdx.y * pstride;
  out += blockIdx.y * ostride;
  const int nd = gprog->ndim;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n1; i += (int64_t)gridDim.x * blockDim.x) {
    double g[BGP_MAX_DIM];
    if (add_prior) kernel_x_gradient<true>(*gprog, 1, x1 + i * nd, x1 + i * nd, g);
    for (int q = 0; q < nd; ++q) {
      double s = 0.0;
      for (int64_t sp = 0; sp < nsplit; ++sp) s += partial[(sp * n1 + i) * nd + q];
      s = scale * s;
      out[i * nd + q] = add_prior ? 2.0 * g[q] + s : s;
    }
  }
}

// the column split of one contraction: nsplit groups of cps XG_TJ-point chunks (~8 CTAs per SM, as matvec_plan)
static int x1_grad_plan(int64_t n1, int64_t n2, int64_t* nsplit_out, int* cps_out) {
  const int64_t row_tiles = (n1 + XG_TI - 1) / XG_TI;
  const int64_t nchunks = (n2 + XG_TJ - 1) / XG_TJ;
  int64_t nsplit = std::max<int64_t>(1, std::min<int64_t>(nchunks, (8 * (int64_t)num_sms() + row_tiles - 1) / row_tiles));
  const int cps = (int)std::max<int64_t>(1, (nchunks + nsplit - 1) / nsplit);
  nsplit = nchunks > 0 ? (nchunks + cps - 1) / cps : 0;
  if (row_tiles > 0x7fffffffLL || nsplit > 65535) { set_error("kmat_x1_gradient_matvec: problem too large for one launch"); return BGP_ERR_INVALID; }
  *nsplit_out = nsplit;
  *cps_out = cps;
  return BGP_OK;
}

// partials of one member's contraction (doubles): nsplit * n1 * nd, nsplit from x1_grad_plan
int64_t x1_grad_partial_size(int64_t n1, int64_t n2, int nd) {
  int64_t nsplit;
  int cps;
  if (n1 <= 0 || x1_grad_plan(n1, n2, &nsplit, &cps) != BGP_OK) return 0;
  return nsplit * n1 * nd;
}

// `members` contractions on the same x1 (n1 points) and x2 (n2 points), in one launch of each kernel: member m uses the
// host program P[m] (device copy dprogs + m), reads V + m * vstride (ldv as above) and writes out + m * ostride (n1 x nd,
// row-major).  The split plan depends on (n1, n2) alone and the evaluator on P[0].shape, so every member's partials
// and their reduction order are those of a one-member call; members whose shapes differ are refused, since the
// specialised and the interpreted evaluators round differently.  x1 / x2 / V / out are device pointers; scratch holds
// members * x1_grad_partial_size(n1, n2, nd) partials.
int kmat_x1_grad_matvec_members(const DevProgram* P, const DevProgram* dprogs, int members, const double* x1,
                                int64_t n1, const double* x2, int64_t n2, const double* V, int64_t ldv,
                                int64_t vstride, double scale, int add_prior, double* out, int64_t ostride,
                                DevBuf<double>& scratch, cudaStream_t s) {
  if (members <= 0) return BGP_OK;
  const int nd = P[0].ndim;
  if (nd > BGP_MAX_DIM) { set_error("input-coordinate gradients support at most %d dimensions (got %d)", BGP_MAX_DIM, nd); return BGP_ERR_INVALID; }
  if (members > 65535) { set_error("kmat_x1_gradient_matvec: more than 65535 members in one launch"); return BGP_ERR_INVALID; }
  for (int m = 1; m < members; ++m)
    if (P[m].shape != P[0].shape || P[m].ndim != nd) {
      set_error("kmat_x1_gradient_matvec: members differ in program structure");
      return BGP_ERR_INVALID;
    }
  if (n1 <= 0) return BGP_OK;
  const unsigned mb = (unsigned)members;
  int64_t nsplit;
  int cps;
  BGP_TRY(x1_grad_plan(n1, n2, &nsplit, &cps));
  const int64_t pstride = nsplit * n1 * nd;
  if (nsplit > 0) {
    BGP_TRY(scratch.reserve((size_t)(pstride * members), s));
    const size_t smem = x1_grad_smem(nd);
    const dim3 grid((unsigned)((n1 + XG_TI - 1) / XG_TI), (unsigned)nsplit, mb);
#define BGP_X1G_LAUNCH(SH)                                                                                   \
  {                                                                                                         \
    cudaFuncSetAttribute(kmat_x1_grad_matvec_kernel<SH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
    kmat_x1_grad_matvec_kernel<SH><<<grid, XG_THREADS, smem, s>>>(dprogs, x1, n1, x2, n2, V, ldv, scratch.p, cps,  \
                                                                  vstride, pstride);                        \
  }
    switch (P[0].shape) {
      case BGP_SHAPE_EXPSQ: BGP_X1G_LAUNCH(BGP_SHAPE_EXPSQ); break;
      case BGP_SHAPE_M32: BGP_X1G_LAUNCH(BGP_SHAPE_M32); break;
      case BGP_SHAPE_M52: BGP_X1G_LAUNCH(BGP_SHAPE_M52); break;
      case BGP_SHAPE_EXP: BGP_X1G_LAUNCH(BGP_SHAPE_EXP); break;
      default: BGP_X1G_LAUNCH(BGP_SHAPE_GENERIC); break;
    }
#undef BGP_X1G_LAUNCH
    BGP_LAUNCH_CHECK();
  }
  const int blocks = (int)std::min<int64_t>((n1 + 127) / 128, 8 * (int64_t)num_sms());
  x1_grad_reduce_kernel<<<dim3((unsigned)blocks, mb), 128, 0, s>>>(dprogs, x1, n1, scratch.p, nsplit, scale, add_prior,
                                                                   out, pstride, ostride);
  BGP_LAUNCH_CHECK();
  return BGP_OK;
}

// out (n1 x nd, row-major) as described above; P is the validated program behind dprog (its shape selects the
// evaluator), x1 / x2 / V / out device pointers.  scratch: the partials (nsplit * n1 * nd doubles).
int kmat_x1_grad_matvec_launch(const DevProgram& P, const DevProgram* dprog, const double* x1, int64_t n1,
                               const double* x2, int64_t n2, const double* V, int64_t ldv, double scale, int add_prior,
                               double* out, DevBuf<double>& scratch, cudaStream_t s) {
  return kmat_x1_grad_matvec_members(&P, dprog, 1, x1, n1, x2, n2, V, ldv, 0, scale, add_prior, out, 0, scratch, s);
}

// ---------------------------------------------------------------------------------------------------------------
// gradient contraction.  Pairs (i, j) with i <= j are evaluated once, as the reference does (kernel_interface.cpp:
// 116-121 evaluates the upper triangle and mirrors), and weighted with A_ij + A_ji (A_ii on the diagonal), where
//     A_ij = ca * alpha_i * alpha_j + cm * M_ij          (grad_log_likelihood: ca = 1, cm = -1, M = K^-1).
// Tiles of 32 x 32 pairs; M's tile and its transposed partner are staged through shared memory so both reads are
// coalesced.  NPMAX is the register budget for the per-parameter accumulators.
// Member blockIdx.z of a batch (bgp_dense_batch_grad_terms) contracts with its own program gprog[z], M + z * mstride,
// alpha + z * astride and writes partial + z * pstride; a single contraction launches one member with zero strides.
// ---------------------------------------------------------------------------------------------------------------
constexpr int GC_T = 32;
constexpr int GC_THREADS = 256;

template <int NPMAX>
__global__ void __launch_bounds__(GC_THREADS) kmat_grad_contract_kernel(const DevProgram* __restrict__ gprog,
                                                                        const unsigned* __restrict__ which,
                                                                        const double* __restrict__ x, int64_t n,
                                                                        const double* __restrict__ M, int64_t ldm,
                                                                        const double* __restrict__ alpha, double ca,
                                                                        double cm, double* __restrict__ partial,
                                                                        int64_t mstride, int64_t astride,
                                                                        int64_t pstride) {
  gprog += blockIdx.z;
  M += blockIdx.z * mstride;
  if (alpha) alpha += blockIdx.z * astride;
  partial += blockIdx.z * pstride;
  __shared__ DevProgram P;
  __shared__ unsigned sw[BGP_MAX_LEAVES * (4 + BGP_MAX_METRIC)];
  __shared__ double tA[GC_T][GC_T + 1], tB[GC_T][GC_T + 1];
  __shared__ double red[32];
  const int np = gprog->n_params_total;
  double acc[NPMAX];
#pragma unroll
  for (int q = 0; q < NPMAX; ++q) acc[q] = 0.0;
  const int64_t nt = (n + GC_T - 1) / GC_T;
  const int64_t bi = blockIdx.y, bj = blockIdx.x;
  const int64_t cta = bi * gridDim.x + bj;
  if (bi <= bj && bi < nt && bj < nt) {
    stage_program(&P, gprog);
    for (int q = threadIdx.x; q < np; q += blockDim.x) sw[q] = which[q];
    const int nd = gprog->ndim;
    const int64_t i0 = bi * GC_T, j0 = bj * GC_T;
    const int ni = (int)min((int64_t)GC_T, n - i0), nj = (int)min((int64_t)GC_T, n - j0);
    // tA[r][c] = M[i0+r][j0+c],  tB[c][r] = M[j0+c][i0+r]   (row-major M with leading dimension ldm; symmetric use)
    for (int t = threadIdx.x; t < GC_T * GC_T; t += GC_THREADS) {
      const int r = t / GC_T, c = t % GC_T;
      tA[r][c] = (r < ni && c < nj) ? M[(i0 + r) * ldm + j0 + c] : 0.0;
      tB[r][c] = (r < nj && c < ni) ? M[(j0 + r) * ldm + i0 + c] : 0.0;
    }
    __syncthreads();
    double g[NPMAX];
    for (int t = threadIdx.x; t < GC_T * GC_T; t += GC_THREADS) {
      const int r = t / GC_T, c = t % GC_T;
      if (r >= ni || c >= nj) continue;
      const int64_t i = i0 + r, j = j0 + c;
      if (i > j) continue;
      double w;
      if (i == j) w = cm * tA[r][c] + (alpha ? ca * alpha[i] * alpha[i] : 0.0);
      else w = cm * (tA[r][c] + tB[c][r]) + (alpha ? 2.0 * ca * alpha[i] * alpha[j] : 0.0);
      kernel_value_grad(P, x + i * nd, x + j * nd, sw, g);
#pragma unroll
      for (int q = 0; q < NPMAX; ++q)
        if (q < np) acc[q] = fma(w, g[q], acc[q]);
    }
  }
  // one partial per (CTA, parameter); CTAs below the diagonal write zeros so the reduction is a plain sum
#pragma unroll
  for (int q = 0; q < NPMAX; ++q) {
    if (q < np) {  // uniform across the CTA
      const double s = block_sum(acc[q], red);
      if (threadIdx.x == 0) partial[cta * np + q] = s;
    }
  }
}

// (member blockIdx.y of a batch: partial + y * pstride, out + y * ostride)
__global__ void grad_contract_reduce_kernel(const double* __restrict__ partial, int64_t nctas, int np,
                                            double* __restrict__ out, int64_t pstride, int64_t ostride) {
  __shared__ double red[32];
  partial += blockIdx.y * pstride;
  out += blockIdx.y * ostride;
  const int q = blockIdx.x;
  double s = 0.0;
  for (int64_t c = threadIdx.x; c < nctas; c += blockDim.x) s += partial[c * np + q];
  s = block_sum(s, red);
  if (threadIdx.x == 0) out[q] = s;
}

// diagA[i] = ca * alpha_i^2 + cm * M_ii  (member blockIdx.y of a batch: M + y * mstride, alpha + y * astride,
// out + y * ostride)
__global__ void grad_diag_kernel(const double* __restrict__ M, int64_t ldm, const double* __restrict__ alpha, double ca,
                                 double cm, int64_t n, double* __restrict__ out, int64_t mstride, int64_t astride,
                                 int64_t ostride) {
  M += blockIdx.y * mstride;
  if (alpha) alpha += blockIdx.y * astride;
  out += blockIdx.y * ostride;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = cm * M[i * ldm + i] + (alpha ? ca * alpha[i] * alpha[i] : 0.0);
}

// g_dev[np] = sum_ij (ca alpha_i alpha_j + cm M_ij) dK_ij/dtheta ; diag_dev[n] (may be null) = diag of that weight matrix.
// `members` contractions of one x in the same three launches: member b uses dprogs[b], M + b * mstride and
// alpha + b * astride, and writes g_dev + b * gstride and diag_dev + b * dstride, exactly as a one-member call computes
// it (the same tiles, NPMAX and reduction order).  All members share np and which_dev; scratch holds
// members * ceil(n / 32)^2 * np partials.
int kmat_grad_contract_members(const DevProgram* dprogs, int np, const unsigned* which_dev, const double* x, int64_t n,
                               const double* M, int64_t ldm, int64_t mstride, const double* alpha, int64_t astride,
                               double ca, double cm, double* g_dev, int64_t gstride, double* diag_dev, int64_t dstride,
                               int members, DevBuf<double>& scratch, cudaStream_t s) {
  if (n <= 0 || members <= 0) return BGP_OK;
  if (np > 64) { set_error("gradient supports at most 64 hyper-parameters"); return BGP_ERR_INVALID; }
  if (members > 65535) { set_error("kmat_grad_contract: more than 65535 members in one launch"); return BGP_ERR_INVALID; }
  const unsigned mb = (unsigned)members;
  if (np > 0) {
    const int64_t nt = (n + GC_T - 1) / GC_T;
    if (nt > 65535) { set_error("kmat_grad_contract: n too large for one launch"); return BGP_ERR_INVALID; }
    const int64_t nctas = nt * nt;
    const int64_t pstride = nctas * np;
    BGP_TRY(scratch.reserve((size_t)(pstride * members), s));
    dim3 grid((unsigned)nt, (unsigned)nt, mb);
    if (np <= 8)
      kmat_grad_contract_kernel<8><<<grid, GC_THREADS, 0, s>>>(dprogs, which_dev, x, n, M, ldm, alpha, ca, cm, scratch.p,
                                                               mstride, astride, pstride);
    else
      kmat_grad_contract_kernel<64><<<grid, GC_THREADS, 0, s>>>(dprogs, which_dev, x, n, M, ldm, alpha, ca, cm, scratch.p,
                                                                mstride, astride, pstride);
    BGP_LAUNCH_CHECK();
    grad_contract_reduce_kernel<<<dim3((unsigned)np, mb), 256, 0, s>>>(scratch.p, nctas, np, g_dev, pstride, gstride);
    BGP_LAUNCH_CHECK();
  }
  if (diag_dev) {
    grad_diag_kernel<<<dim3((unsigned)std::min<int64_t>((n + 255) / 256, 1184), mb), 256, 0, s>>>(
        M, ldm, alpha, ca, cm, n, diag_dev, mstride, astride, dstride);
    BGP_LAUNCH_CHECK();
  }
  return BGP_OK;
}
int kmat_grad_contract_launch(const DevProgram* dprog, int nd, int np, const unsigned* which_dev, const double* x,
                              int64_t n, const double* M, int64_t ldm, const double* alpha, double ca, double cm,
                              double* g_dev, double* diag_dev, DevBuf<double>& scratch, cudaStream_t s) {
  (void)nd;
  return kmat_grad_contract_members(dprog, np, which_dev, x, n, M, ldm, 0, alpha, 0, ca, cm, g_dev, 0, diag_dev, 0, 1,
                                    scratch, s);
}

// One hyper-parameter's plane of the kernel gradient, out[i * ldo + j] = d k(x_i, x_j) / d theta_p (n x n), for
// GP.fisher_information's kernel rows: kmat_gradient_kernel interleaves all P planes, which would make the Fisher pass's
// memory grow with P.  Every entry evaluates the pair as (x_min(i,j), x_max(i,j)), so the plane is exactly symmetric, with
// parameter p the only active one.  One thread per entry along j: the stores are coalesced, and the ~2x evaluations are
// noise beside the O(n^3) products that consume the plane.
// Member blockIdx.y of a batch evaluates with gprog + y and writes its plane at out + y * ostride.
template <int NPMAX>
__global__ void __launch_bounds__(256) kmat_gradient_plane_kernel(const DevProgram* __restrict__ gprog, int p,
                                                                  const double* __restrict__ x, int64_t n,
                                                                  double* __restrict__ out, int64_t ldo,
                                                                  int64_t ostride) {
  gprog += blockIdx.y;
  out += blockIdx.y * ostride;
  __shared__ DevProgram P;
  __shared__ unsigned sw[BGP_MAX_LEAVES * (4 + BGP_MAX_METRIC)];
  stage_program(&P, gprog);
  const int np = gprog->n_params_total;
  for (int q = threadIdx.x; q < np; q += blockDim.x) sw[q] = (q == p) ? 1u : 0u;
  __syncthreads();
  const int nd = P.ndim;
  double g[NPMAX];
  const int64_t total = n * n;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / n, j = t - i * n;
    const int64_t a = i < j ? i : j, b = i < j ? j : i;
    kernel_value_grad(P, x + a * nd, x + b * nd, sw, g);
    double v = 0.0;
#pragma unroll
    for (int q = 0; q < NPMAX; ++q)
      if (q == p) v = g[q];
    out[i * ldo + j] = v;
  }
}

// `members` planes of one x in one launch: member b evaluates with dprogs[b] and writes out + b * ostride, each entry
// exactly as a one-member call computes it.  All members share np and p.
int kmat_gradient_plane_members(const DevProgram* dprogs, int np, int p, const double* x, int64_t n, double* out,
                                int64_t ldo, int64_t ostride, int members, cudaStream_t s) {
  if (n <= 0 || members <= 0) return BGP_OK;
  if (np > 64) { set_error("gradient supports at most 64 hyper-parameters"); return BGP_ERR_INVALID; }
  if (p < 0 || p >= np) { set_error("gradient plane %d out of range (%d parameters)", p, np); return BGP_ERR_INVALID; }
  if (members > 65535) { set_error("gradient plane: more than 65535 members in one launch"); return BGP_ERR_INVALID; }
  const dim3 grid((unsigned)std::min<int64_t>((n * n + 255) / 256, 16 * (int64_t)num_sms()), (unsigned)members);
  if (np <= 8) kmat_gradient_plane_kernel<8><<<grid, 256, 0, s>>>(dprogs, p, x, n, out, ldo, ostride);
  else kmat_gradient_plane_kernel<64><<<grid, 256, 0, s>>>(dprogs, p, x, n, out, ldo, ostride);
  BGP_LAUNCH_CHECK();
  return BGP_OK;
}
int kmat_gradient_plane_launch(const DevProgram* dprog, int np, int p, const double* x, int64_t n, double* out,
                               int64_t ldo, cudaStream_t s) {
  return kmat_gradient_plane_members(dprog, np, p, x, n, out, ldo, 0, 1, s);
}

// ---------------------------------------------------------------------------------------------------------------
// Slab gradient contraction (bgp_hodlr_grad_terms at large n, which never holds all of K^-1): for a slab
// W = K^-1 E_J of columns J = [j0, j0 + nc) (n x nc, column-major, W[(j - j0) n + i] = (K^-1)_ij),
//     g_p += sum_{i, j in J} (u_i v_j - W_ij) dK_ij/dtheta_p,
// u = v = alpha for grad_log_likelihood.  bgp_hodlr_loo_terms passes u = beta, v = alpha and W = K^-1 diag(c) K^-1 E_J:
// summed over every ordered pair against a symmetric dK, u_i v_j gives what the symmetrised 1/2 (u_i v_j + v_i u_j)
// gives.
// Every ordered pair is evaluated (george's einsum over all (i, j)): the symmetric weighting of
// kmat_grad_contract_kernel would need rows of K^-1 from two slabs.  One thread per row i; the coordinates and alpha of
// a 32-column j-tile are staged in shared memory and W is read coalesced along i.  CTA (tile t, split s) covers rows
// [s GS_ROWS, (s + 1) GS_ROWS) of tile t and writes one partial per parameter; grad_slab_reduce_kernel sums the splits
// in order into the tile's slot of a (ceil(n / 32) x P) array, and grad_contract_reduce_kernel sums the tiles in order
// once every slab is done.  The split plan and the tile boundaries depend only on n (slabs start at multiples of 64),
// so g does not depend on the slab width, and no atomics: two identical calls return the same bits.
// A column window [jlo, jhi) restricts the sum to j in the window (a shard of a sharded factorisation owns the columns
// of its rows, bgp_hodlr_grad_terms_local_dev): a tile that straddles a window edge contributes only its columns inside
// it (the others carry weight 0, set where alpha_j is staged, so the inner loop and its registers are those of the
// unrestricted kernel), the tile boundaries stay global multiples of 32, and the window [0, n) is the unrestricted sum,
// bit for bit.
// ---------------------------------------------------------------------------------------------------------------
constexpr int GS_TJ = 32;          // columns per j-tile
constexpr int GS_THREADS = 256;
constexpr int64_t GS_ROWS = 1024;  // rows per i-split
// x_j staging (inputs of up to 128 dimensions): with the ~12 KB of static shared memory it stays under the default
// 48 KB per CTA; wider inputs read x_j from global memory
constexpr size_t GS_SMEM_CAP = 32 * 1024;
constexpr int GS_WARPS = GS_THREADS / 32;

// XSHAPE >= 0 (GP.grad_log_likelihood_x, bgp_hodlr_grad_x_terms): the same pass also contracts the input gradient of
// each of the tile's columns j,
//     xpart[((tile * nsplit + split) * GS_TJ + c) * nd + q] = sum_{i in split} w_ij d k(x_j, x_i) / d x_jq,
// with w_ij = u_i v_j - W_ij the weight of the parameter contraction and the evaluator of kmat_x1_grad_matvec_kernel for
// shape XSHAPE (the arguments swapped, x_j first, so a non-stationary kernel is differentiated in x_j).  Each warp sums
// its 32 rows of a column with warp_sum and adds the sum to its own slot in shared memory; the CTA then adds the warps'
// slots in warp order.  A NULL `which` skips the parameter contraction.  Needs nd <= BGP_MAX_DIM and staged x_j.
template <int NPMAX, int XSHAPE = -1>
__global__ void __launch_bounds__(GS_THREADS) kmat_grad_slab_kernel(const DevProgram* __restrict__ gprog,
                                                                    const unsigned* __restrict__ which,
                                                                    const double* __restrict__ x, int64_t n,
                                                                    const double* __restrict__ W, int64_t j0,
                                                                    int64_t nc, int64_t jlo, int64_t jhi,
                                                                    const double* __restrict__ u,
                                                                    const double* __restrict__ v, int stage_x,
                                                                    double* __restrict__ partial,
                                                                    double* __restrict__ xpart = nullptr) {
  extern __shared__ double sxj[];  // GS_TJ x nd coordinates of the tile's columns (stage_x)
  __shared__ DevProgram P;
  __shared__ unsigned sw[BGP_MAX_LEAVES * (4 + BGP_MAX_METRIC)];
  __shared__ double saj[GS_TJ];
  __shared__ double red[32];
  const int np = (XSHAPE >= 0 && !which) ? 0 : gprog->n_params_total, nd = gprog->ndim;
  const int64_t jt = j0 + (int64_t)blockIdx.x * GS_TJ;  // first column of the tile
  const int nj = (int)min((int64_t)GS_TJ, j0 + nc - jt);
  const int64_t r0 = (int64_t)blockIdx.y * GS_ROWS, r1 = min(n, r0 + GS_ROWS);
  stage_program(&P, gprog);
  for (int q = threadIdx.x; q < np; q += blockDim.x) sw[q] = which[q];
  // a column outside the window gets weight 0 (v_j staged as 0, and its W column is zero: the identity is placed in
  // the window only), so it adds exactly nothing, and the loop below carries no window bounds
  if (threadIdx.x < nj) {
    const int64_t j = jt + threadIdx.x;
    saj[threadIdx.x] = (j >= jlo && j < jhi) ? v[j] : 0.0;
  }
  if (stage_x)
    for (int t = threadIdx.x; t < nj * nd; t += GS_THREADS) sxj[t] = x[jt * nd + t];
  __syncthreads();
  const double* Wt = W + (jt - j0) * n;
  double acc[NPMAX], g[NPMAX];
#pragma unroll
  for (int q = 0; q < NPMAX; ++q) acc[q] = 0.0;
  if constexpr (XSHAPE < 0) {
    for (int64_t i = r0 + threadIdx.x; i < r1; i += GS_THREADS) {
      const double ai = u[i];
      const double* xi = x + i * nd;
      for (int c = 0; c < nj; ++c) {
        const double w = ai * saj[c] - Wt[(int64_t)c * n + i];
        kernel_value_grad(P, xi, stage_x ? sxj + c * nd : x + (jt + c) * nd, sw, g);
#pragma unroll
        for (int q = 0; q < NPMAX; ++q)
          if (q < np) acc[q] = fma(w, g[q], acc[q]);
      }
    }
  } else {
    using Eval = X1GradEval<XSHAPE>;
    constexpr int NDMAX = Eval::type::NDMAX;
    const typename Eval::type fx = Eval::make(&P);
    double* wdx = sxj + GS_TJ * nd;  // GS_WARPS x GS_TJ x nd: warp w's sums of column c
    for (int t = threadIdx.x; t < GS_WARPS * GS_TJ * nd; t += GS_THREADS) wdx[t] = 0.0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // every lane runs every row step (a lane past r1 adds zeros) so that the warp sums see the whole warp; the
    // parameter sums of a live row run in the order of the unflagged kernel, so they keep its bits
    for (int64_t ib = r0; ib < r1; ib += GS_THREADS) {
      const int64_t i = ib + threadIdx.x;
      const bool live = i < r1;
      const double ai = live ? u[i] : 0.0;
      const double* xi = x + (live ? i : r0) * nd;
      for (int c = 0; c < nj; ++c) {
        double gx[NDMAX];
        double w = 0.0;
        if (live) {
          w = ai * saj[c] - Wt[(int64_t)c * n + i];
          if (np) {
            kernel_value_grad(P, xi, sxj + c * nd, sw, g);
#pragma unroll
            for (int q = 0; q < NPMAX; ++q)
              if (q < np) acc[q] = fma(w, g[q], acc[q]);
          }
          fx(sxj + c * nd, xi, gx);
        } else {
#pragma unroll
          for (int q = 0; q < NDMAX; ++q) gx[q] = 0.0;
        }
#pragma unroll
        for (int q = 0; q < NDMAX; ++q) {
          if (q < nd) {  // uniform across the warp
            const double s = warp_sum(w * gx[q]);
            if (lane == 0) wdx[(warp * GS_TJ + c) * nd + q] += s;
          }
        }
      }
    }
  }
  // one partial per (tile, split, parameter)
#pragma unroll
  for (int q = 0; q < NPMAX; ++q) {
    if (q < np) {  // uniform across the CTA
      const double s = block_sum(acc[q], red);
      if (threadIdx.x == 0) partial[((int64_t)blockIdx.x * gridDim.y + blockIdx.y) * np + q] = s;
    }
  }
  if constexpr (XSHAPE >= 0) {
    __syncthreads();
    const double* wdx = sxj + GS_TJ * nd;
    double* out = xpart + ((int64_t)blockIdx.x * gridDim.y + blockIdx.y) * GS_TJ * nd;
    for (int t = threadIdx.x; t < nj * nd; t += GS_THREADS) {
      double s = wdx[t];
      for (int w = 1; w < GS_WARPS; ++w) s += wdx[w * GS_TJ * nd + t];
      out[t] = s;
    }
  }
}

// dx[j * nd + q] = sum_s xpart[((tile * nsplit + s) * GS_TJ + c) * nd + q], s ascending, for the columns
// j = j0 + tile * GS_TJ + c of one slab that lie in the window [jlo, jhi) (no other row is written)
__global__ void grad_slab_x_reduce_kernel(const double* __restrict__ xpart, int64_t nsplit, int64_t j0, int64_t nc,
                                          int64_t jlo, int64_t jhi, int nd, double* __restrict__ dx) {
  const int64_t total = nc * nd;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = t / nd, q = t - k * nd, j = j0 + k;
    if (j < jlo || j >= jhi) continue;
    const int64_t tile = k / GS_TJ, c = k - tile * GS_TJ;
    double s = 0.0;
    for (int64_t sp = 0; sp < nsplit; ++sp) s += xpart[((tile * nsplit + sp) * GS_TJ + c) * nd + q];
    dx[j * nd + q] = s;
  }
}

// tile_part[t * np + q] = sum_s partial[(t * nsplit + s) * np + q], s ascending, for the ntile tiles of one slab
__global__ void grad_slab_reduce_kernel(const double* __restrict__ partial, int64_t nsplit, int64_t ntile, int np,
                                        double* __restrict__ tile_part) {
  const int64_t total = ntile * np;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t tile = t / np, q = t - tile * np;
    double s = 0.0;
    for (int64_t sp = 0; sp < nsplit; ++sp) s += partial[(tile * nsplit + sp) * np + q];
    tile_part[t] = s;
  }
}

// diag[j] = u_j v_j - W_jj for j in [j0, j0 + nc) inside the window [jlo, jhi) (no other entry is written): the
// product and the difference rounded separately (no contraction into an FMA), as alpha**2 - diag(K^-1) is on the host
__global__ void grad_slab_diag_kernel(const double* __restrict__ W, int64_t n, int64_t j0, int64_t nc, int64_t jlo,
                                      int64_t jhi, const double* __restrict__ u, const double* __restrict__ v,
                                      double* __restrict__ diag) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nc; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t j = j0 + k;
    if (j >= jlo && j < jhi) diag[j] = __dsub_rn(__dmul_rn(u[j], v[j]), W[k * n + j]);
  }
}

// doubles of per-slab partials for slabs of up to c columns of an n-row K^-1
int64_t grad_slab_partial_size(int64_t n, int64_t c, int np) {
  return ((n + GS_ROWS - 1) / GS_ROWS) * ((c + GS_TJ - 1) / GS_TJ) * std::max(np, 1);
}
// doubles of per-tile partials (all slabs) for an n-row K^-1
int64_t grad_slab_tile_size(int64_t n, int np) { return ((n + GS_TJ - 1) / GS_TJ) * std::max(np, 1); }

// One slab (j0 a multiple of 32) restricted to the columns [jlo, jhi): its tiles' partials into
// tile_part + (j0 / 32) * np, and diag[j] for j in [j0, j0 + nc) and in the window when diag_dev is set.  Passing
// u = v = alpha is the contraction of grad_log_likelihood, bit for bit.
// partial: grad_slab_partial_size(n, nc, np) doubles.
int kmat_grad_slab_launch(const DevProgram* dprog, int nd, int np, const unsigned* which_dev, const double* x, int64_t n,
                          const double* W, int64_t j0, int64_t nc, int64_t jlo, int64_t jhi, const double* u,
                          const double* v, double* partial, double* tile_part, double* diag_dev, cudaStream_t s) {
  if (nc <= 0) return BGP_OK;
  if (np > 64) { set_error("gradient supports at most 64 hyper-parameters"); return BGP_ERR_INVALID; }
  if (j0 % GS_TJ) { set_error("internal: slab start %lld is not a multiple of %d", (long long)j0, GS_TJ); return BGP_ERR_INVALID; }
  if (np > 0) {
    const int64_t nsplit = (n + GS_ROWS - 1) / GS_ROWS, ntile = (nc + GS_TJ - 1) / GS_TJ;
    if (nsplit > 65535 || ntile > 0x7fffffffLL) { set_error("kmat_grad_slab: n too large for one launch"); return BGP_ERR_INVALID; }
    const size_t sbytes = sizeof(double) * (size_t)GS_TJ * nd;
    const int stage_x = sbytes <= GS_SMEM_CAP ? 1 : 0;
    const size_t smem = stage_x ? sbytes : 0;
    const dim3 grid((unsigned)ntile, (unsigned)nsplit);
    if (np <= 8)
      kmat_grad_slab_kernel<8><<<grid, GS_THREADS, smem, s>>>(dprog, which_dev, x, n, W, j0, nc, jlo, jhi, u, v,
                                                               stage_x, partial);
    else
      kmat_grad_slab_kernel<64><<<grid, GS_THREADS, smem, s>>>(dprog, which_dev, x, n, W, j0, nc, jlo, jhi, u, v,
                                                                stage_x, partial);
    BGP_LAUNCH_CHECK();
    const int64_t total = ntile * np;
    grad_slab_reduce_kernel<<<(unsigned)std::min<int64_t>((total + 255) / 256, 8 * (int64_t)num_sms()), 256, 0, s>>>(
        partial, nsplit, ntile, np, tile_part + (j0 / GS_TJ) * np);
    BGP_LAUNCH_CHECK();
  }
  if (diag_dev) {
    grad_slab_diag_kernel<<<(unsigned)std::min<int64_t>((nc + 255) / 256, 1184), 256, 0, s>>>(W, n, j0, nc, jlo, jhi,
                                                                                              u, v, diag_dev);
    BGP_LAUNCH_CHECK();
  }
  return BGP_OK;
}

// doubles of per-slab input-gradient partials for slabs of up to c columns of an n-row K^-1, nd-dimensional inputs
int64_t grad_slab_x_partial_size(int64_t n, int64_t c, int nd) {
  return ((n + GS_ROWS - 1) / GS_ROWS) * ((c + GS_TJ - 1) / GS_TJ) * GS_TJ * std::max(nd, 1);
}

// kmat_grad_slab_launch with the input gradient of the slab's columns in the same pass (bgp_hodlr_grad_x_terms):
// the parameter partials, tile_part and diag exactly as kmat_grad_slab_launch writes them with u = v = alpha (the same
// kernel body, bit for bit), and dx_dev[j * nd + q] = sum_i (alpha_i alpha_j - W_ij) d k(x_j, x_i) / d x_jq for the
// columns j of the slab in [jlo, jhi), summed over the row splits in order: dx_j depends on n alone, not on the slab
// width.  which_dev NULL (np 0) skips the parameter contraction.  shape: the program's shape (it selects the evaluator,
// as in kmat_x1_grad_matvec_members); nd <= BGP_MAX_DIM.  xpart: grad_slab_x_partial_size(n, nc, nd) doubles.
int kmat_grad_x_slab_launch(const DevProgram* dprog, int shape, int nd, int np, const unsigned* which_dev,
                            const double* x, int64_t n, const double* W, int64_t j0, int64_t nc, int64_t jlo,
                            int64_t jhi, const double* alpha, double* partial, double* tile_part, double* xpart,
                            double* diag_dev, double* dx_dev, cudaStream_t s) {
  if (nc <= 0) return BGP_OK;
  if (!which_dev) np = 0;
  if (np > 64) { set_error("gradient supports at most 64 hyper-parameters"); return BGP_ERR_INVALID; }
  if (nd > BGP_MAX_DIM) { set_error("input-coordinate gradients support at most %d dimensions (got %d)", BGP_MAX_DIM, nd); return BGP_ERR_INVALID; }
  if (j0 % GS_TJ) { set_error("internal: slab start %lld is not a multiple of %d", (long long)j0, GS_TJ); return BGP_ERR_INVALID; }
  const int64_t nsplit = (n + GS_ROWS - 1) / GS_ROWS, ntile = (nc + GS_TJ - 1) / GS_TJ;
  if (nsplit > 65535 || ntile > 0x7fffffffLL) { set_error("kmat_grad_slab: n too large for one launch"); return BGP_ERR_INVALID; }
  const size_t smem = sizeof(double) * (size_t)(1 + GS_WARPS) * GS_TJ * nd;  // x_j staged, then the warps' sums
  const dim3 grid((unsigned)ntile, (unsigned)nsplit);
  const unsigned* which = np ? which_dev : nullptr;
#define BGP_GXS_LAUNCH(NPM, SH)                                                                                  \
  kmat_grad_slab_kernel<NPM, SH><<<grid, GS_THREADS, smem, s>>>(dprog, which, x, n, W, j0, nc, jlo, jhi, alpha, alpha, \
                                                                1, partial, xpart)
#define BGP_GXS_SHAPES(NPM)                                                   \
  switch (shape) {                                                            \
    case BGP_SHAPE_EXPSQ: BGP_GXS_LAUNCH(NPM, BGP_SHAPE_EXPSQ); break;        \
    case BGP_SHAPE_M32: BGP_GXS_LAUNCH(NPM, BGP_SHAPE_M32); break;            \
    case BGP_SHAPE_M52: BGP_GXS_LAUNCH(NPM, BGP_SHAPE_M52); break;            \
    case BGP_SHAPE_EXP: BGP_GXS_LAUNCH(NPM, BGP_SHAPE_EXP); break;            \
    default: BGP_GXS_LAUNCH(NPM, BGP_SHAPE_GENERIC); break;                   \
  }
  if (np <= 8) {
    BGP_GXS_SHAPES(8)
  } else {
    BGP_GXS_SHAPES(64)
  }
#undef BGP_GXS_SHAPES
#undef BGP_GXS_LAUNCH
  BGP_LAUNCH_CHECK();
  if (np > 0) {
    const int64_t total = ntile * np;
    grad_slab_reduce_kernel<<<(unsigned)std::min<int64_t>((total + 255) / 256, 8 * (int64_t)num_sms()), 256, 0, s>>>(
        partial, nsplit, ntile, np, tile_part + (j0 / GS_TJ) * np);
    BGP_LAUNCH_CHECK();
  }
  grad_slab_x_reduce_kernel<<<(unsigned)std::min<int64_t>((nc * nd + 255) / 256, 8 * (int64_t)num_sms()), 256, 0, s>>>(
      xpart, nsplit, j0, nc, jlo, jhi, nd, dx_dev);
  BGP_LAUNCH_CHECK();
  if (diag_dev) {
    grad_slab_diag_kernel<<<(unsigned)std::min<int64_t>((nc + 255) / 256, 1184), 256, 0, s>>>(W, n, j0, nc, jlo, jhi,
                                                                                              alpha, alpha, diag_dev);
    BGP_LAUNCH_CHECK();
  }
  return BGP_OK;
}

// A (n x n, in place) = alpha alpha^T - A: K^-1 becomes the weight of the log-likelihood's gradient, the product and the
// difference rounded separately, as np.outer(alpha, alpha) - K^-1 on the host
__global__ void grad_x_form_a_kernel(double* __restrict__ A, int64_t n, const double* __restrict__ alpha) {
  const int64_t total = n * n;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t j = t / n, i = t - j * n;
    A[t] = __dsub_rn(__dmul_rn(alpha[i], alpha[j]), A[t]);
  }
}

// The resident input gradient of bgp_dense_grad_x_terms and bgp_hodlr_grad_x_terms: with Kinv (n x n) = K^-1,
//     dx[i * nd + q] = sum_j (alpha_i alpha_j - K^-1_ji) d k(x_i, x_j) / d x_iq,
// Kinv overwritten by alpha alpha^T - K^-1, then contracted by the x-gradient matvec of GP.grad_predict with V = that
// matrix (column i holds the weights of point i).  P: the host program (its shape selects the evaluator).
int grad_x_resident_launch(const DevProgram& P, const DevProgram* dprog, const double* x, int64_t n, double* Kinv,
                           const double* alpha, double* dx_dev, DevBuf<double>& scratch, cudaStream_t s) {
  if (n <= 0) return BGP_OK;
  grad_x_form_a_kernel<<<(unsigned)std::min<int64_t>((n * n + 255) / 256, 16 * (int64_t)num_sms()), 256, 0, s>>>(Kinv, n,
                                                                                                             alpha);
  BGP_LAUNCH_CHECK();
  return kmat_x1_grad_matvec_launch(P, dprog, x, n, x, n, Kinv, n, 1.0, 0, dx_dev, scratch, s);
}

// g_dev[q] = sum_t tile_part[t * np + q] over the tiles that meet the columns [jlo, jhi) (all ceil(n / 32) tiles for
// [0, n)), in a fixed order that depends only on the window
int kmat_grad_slab_finish(int np, int64_t jlo, int64_t jhi, const double* tile_part, double* g_dev, cudaStream_t s) {
  if (np <= 0) return BGP_OK;
  const int64_t t0 = jlo / GS_TJ, t1 = (jhi + GS_TJ - 1) / GS_TJ;
  grad_contract_reduce_kernel<<<dim3((unsigned)np, 1), 256, 0, s>>>(tile_part + t0 * np, t1 - t0, np, g_dev, 0, 0);
  BGP_LAUNCH_CHECK();
  return BGP_OK;
}

// `members` identity matrices of order n, back to back (member stride n^2; column-major == row-major)
__global__ void fill_identity_kernel(double* __restrict__ A, int64_t n, int64_t total) {
  const int64_t nn = n * n;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t u = t % nn;
    A[t] = (u / n == u % n) ? 1.0 : 0.0;
  }
}
int fill_identity_members(double* A, int64_t n, int members, cudaStream_t s) {
  const int64_t total = n * n * members;
  fill_identity_kernel<<<(unsigned)std::min<int64_t>((total + 255) / 256, 16 * (int64_t)num_sms()), 256, 0, s>>>(A, n, total);
  BGP_LAUNCH_CHECK();
  return BGP_OK;
}
int fill_identity_launch(double* A, int64_t n, cudaStream_t s) { return fill_identity_members(A, n, 1, s); }

// ---------------------------------------------------------------------------------------------------------------
// Leave-one-out cross-validation (bgp_dense_loo_terms, bgp_hodlr_loo_terms; Rasmussen & Williams, GPML eqs. 5.10-5.13):
// with alpha = K^-1 r and d = diag(K^-1), the gradient of L_loo = sum_i [1/2 log d_i - alpha_i^2 / (2 d_i)] + const
// contracts A = 1/2 (beta alpha^T + alpha beta^T) - K^-1 diag(c) K^-1 with dK, where
//     q_i = alpha_i / d_i,   beta = K^-1 q,   c_i = (1 + alpha_i q_i) / (2 d_i).
// ---------------------------------------------------------------------------------------------------------------
// (member blockIdx.y of a batch: every vector + y * n)
__global__ void loo_weights_kernel(const double* __restrict__ alpha, const double* __restrict__ d, int64_t n,
                                   double* __restrict__ q, double* __restrict__ c) {
  const int64_t m = (int64_t)blockIdx.y * n;
  alpha += m; d += m; q += m; c += m;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const double qi = alpha[i] / d[i];
    q[i] = qi;
    c[i] = (1.0 + alpha[i] * qi) / (2.0 * d[i]);
  }
}
// `members` vectors of n back to back (member stride n); a single call passes one member
int loo_weights_members(const double* alpha, const double* d, int64_t n, double* q, double* c, int members,
                        cudaStream_t s) {
  if (n <= 0 || members <= 0) return BGP_OK;
  loo_weights_kernel<<<dim3((unsigned)std::min<int64_t>((n + 255) / 256, 1184), (unsigned)members), 256, 0, s>>>(
      alpha, d, n, q, c);
  BGP_LAUNCH_CHECK();
  return BGP_OK;
}
int loo_weights_launch(const double* alpha, const double* d, int64_t n, double* q, double* c, cudaStream_t s) {
  return loo_weights_members(alpha, d, n, q, c, 1, s);
}

// X (n x ncols, column-major ldx): row i scaled by w_i, or by sqrt(w_i) with `sqrt_w` (member blockIdx.y of a batch:
// X + y * xstride, w + y * wstride)
__global__ void scale_rows_kernel(double* __restrict__ X, int64_t n, int64_t ncols, int64_t ldx,
                                  const double* __restrict__ w, int sqrt_w, int64_t xstride, int64_t wstride) {
  X += blockIdx.y * xstride;
  w += blockIdx.y * wstride;
  const int64_t total = n * ncols;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t j = t / n, i = t - j * n;
    X[j * ldx + i] *= sqrt_w ? sqrt(w[i]) : w[i];
  }
}
int scale_rows_members(double* X, int64_t n, int64_t ncols, int64_t ldx, const double* w, bool sqrt_w, int members,
                       int64_t xstride, int64_t wstride, cudaStream_t s) {
  const int64_t total = n * ncols;
  if (total <= 0 || members <= 0) return BGP_OK;
  scale_rows_kernel<<<dim3((unsigned)std::min<int64_t>((total + 255) / 256, 16 * (int64_t)num_sms()), (unsigned)members),
                      256, 0, s>>>(X, n, ncols, ldx, w, sqrt_w ? 1 : 0, xstride, wstride);
  BGP_LAUNCH_CHECK();
  return BGP_OK;
}
int scale_rows_launch(double* X, int64_t n, int64_t ncols, int64_t ldx, const double* w, bool sqrt_w, cudaStream_t s) {
  return scale_rows_members(X, n, ncols, ldx, w, sqrt_w, 1, 0, 0, s);
}

// The gradient needs every d_j > 0 (c and sqrt(c) are formed from it); a loose-tolerance HODLR matrix, or rounding of
// a nearly singular K, can break that.  BGP_ERR_INVALID names the first offending point.
int loo_check_diag(const double* d, int64_t n) {
  for (int64_t j = 0; j < n; ++j)
    if (!(d[j] > 0.0) || !std::isfinite(d[j])) {
      set_error("leave-one-out: diag(K^-1) at point %lld is %g, not a finite positive number", (long long)j, d[j]);
      return BGP_ERR_INVALID;
    }
  return BGP_OK;
}

// d[j0 + k] = W[k * ldw + j0 + k] for k < nc: the diagonal entries of the slab W = K^-1 E_J, J = [j0, j0 + nc)
// (member blockIdx.y of a batch: W + y * wstride, d + y * dstride)
__global__ void slab_diag_kernel(const double* __restrict__ W, int64_t ldw, int64_t j0, int64_t nc,
                                 double* __restrict__ d, int64_t wstride, int64_t dstride) {
  W += blockIdx.y * wstride;
  d += blockIdx.y * dstride;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nc; k += (int64_t)gridDim.x * blockDim.x)
    d[j0 + k] = W[k * ldw + j0 + k];
}
int slab_diag_members(const double* W, int64_t ldw, int64_t j0, int64_t nc, double* d, int members, int64_t wstride,
                      int64_t dstride, cudaStream_t s) {
  if (nc <= 0 || members <= 0) return BGP_OK;
  slab_diag_kernel<<<dim3((unsigned)std::min<int64_t>((nc + 255) / 256, 1184), (unsigned)members), 256, 0, s>>>(
      W, ldw, j0, nc, d, wstride, dstride);
  BGP_LAUNCH_CHECK();
  return BGP_OK;
}
int slab_diag_launch(const double* W, int64_t ldw, int64_t j0, int64_t nc, double* d, cudaStream_t s) {
  return slab_diag_members(W, ldw, j0, nc, d, 1, 0, 0, s);
}

// ---------------------------------------------------------------------------------------------------------------
// Predictive variance / covariance (GP.predict with return_var / return_cov; bgp_dense_predict, bgp_hodlr_predict).
// The solvers stream the test points in column chunks: B = K(x, x*_chunk) (N x c), W = K^-1 B (HODLR) or L^-1 B
// (dense, W = B in place), then
//   variance    var_j = k(x*_j, x*_j) - sum_i B_ij W_ij      (two passes: per-CTA partials, fixed-order finish)
//   covariance  C -= W^T B  on the tensor pipe, split over K = N into zeroed slices added in a fixed order.
// No atomics anywhere: two identical calls return bit-identical results.
// ---------------------------------------------------------------------------------------------------------------
constexpr int PV_THREADS = 256;
constexpr int64_t PV_MIN_ROWS = 1024;       // rows of one column per CTA, at least
constexpr int64_t PREDICT_BUDGET = 1 << 27; // doubles (1 GiB) of per-chunk workspace / covariance slices

// Columns per chunk: as many N-row columns as fit in PREDICT_BUDGET, at least 64, a multiple of `multiple`.
// BGP_PREDICT_CHUNK=<c> (read at every call, like BGP_DENSE_OB) forces c, rounded up to `multiple`; tests use it to run
// many chunks with a ragged tail at small sizes.
int64_t predict_chunk_cols(int64_t n, int64_t multiple) {
  int64_t c = std::max<int64_t>(64, (PREDICT_BUDGET / std::max<int64_t>(n, 1)) / 64 * 64);
  if (const char* e = getenv("BGP_PREDICT_CHUNK")) {
    const long v = atol(e);
    if (v >= 1) c = v;
  }
  return (c + multiple - 1) / multiple * multiple;
}

// partial[j * nsplit + b] = sum over the rows of split b of B[j*ldb + i] * W[j*ldw + i]; grid (c, nsplit, members):
// member z reads B and W + z * mstride and writes partial + z * c * nsplit
__global__ void __launch_bounds__(PV_THREADS) predict_var_partial_kernel(const double* __restrict__ B, int64_t ldb,
                                                                         const double* __restrict__ W, int64_t ldw,
                                                                         int64_t n, int64_t rows_per_split,
                                                                         double* __restrict__ partial, int64_t mstride) {
  __shared__ double red[32];
  B += blockIdx.z * mstride;
  W += blockIdx.z * mstride;
  partial += (int64_t)blockIdx.z * gridDim.x * gridDim.y;
  const int64_t j = blockIdx.x;
  const int64_t r0 = (int64_t)blockIdx.y * rows_per_split, r1 = min(n, r0 + rows_per_split);
  const double* b = B + j * ldb;
  const double* w = W + j * ldw;
  double s = 0.0;
  for (int64_t i = r0 + threadIdx.x; i < r1; i += PV_THREADS) s = fma(b[i], w[i], s);
  s = block_sum(s, red);
  if (threadIdx.x == 0) partial[j * gridDim.y + blockIdx.y] = s;
}

// var[j] = kdiag[j] - sum_b partial[j * nsplit + b], b ascending (member blockIdx.y of a batch: partial + y * c * nsplit,
// kdiag and var + y * vstride)
__global__ void predict_var_finish_kernel(const double* __restrict__ partial, int nsplit, const double* __restrict__ kdiag,
                                          int64_t c, double* __restrict__ var, int64_t vstride) {
  partial += blockIdx.y * c * nsplit;
  kdiag += blockIdx.y * vstride;
  var += blockIdx.y * vstride;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < c; j += (int64_t)gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int b = 0; b < nsplit; ++b) s += partial[j * nsplit + b];
    var[j] = kdiag[j] - s;
  }
}

// the row split of a variance chunk of c columns of n rows: nsplit groups of `rows` rows, one partial per (column, group)
static void predict_var_plan(int64_t n, int64_t c, int64_t* nsplit_out, int64_t* rows_out) {
  int64_t nsplit = std::max<int64_t>(1, std::min<int64_t>((4 * (int64_t)num_sms() + c - 1) / c, (n + PV_MIN_ROWS - 1) / PV_MIN_ROWS));
  const int64_t rows = (n + nsplit - 1) / nsplit;
  *nsplit_out = (n + rows - 1) / rows;
  *rows_out = rows;
}
// doubles of variance partials per member for a chunk of c columns
int64_t predict_var_partial_size(int64_t n, int64_t c) {
  if (c <= 0) return 0;
  int64_t nsplit, rows;
  predict_var_plan(n, c, &nsplit, &rows);
  return c * nsplit;
}

// var (c) = kdiag - colsum(B .* W); B, W: n x c column-major, leading dimensions ldb and ldw (B == W for the dense
// solver; a HODLR shard's B holds its own rows only, W all N).
// `members` > 1: member b reads B and W + b * mstride and writes var + b * vstride from kdiag + b * vstride, in the
// same two launches; scratch holds members * predict_var_partial_size(n, c).
int predict_var_batch_launch(const double* B, int64_t ldb, const double* W, int64_t ldw, int64_t n, int64_t c,
                             const double* kdiag, double* var, int members, int64_t mstride, int64_t vstride,
                             DevBuf<double>& scratch, cudaStream_t s) {
  if (c <= 0 || members <= 0) return BGP_OK;
  int64_t nsplit, rows;
  predict_var_plan(n, c, &nsplit, &rows);
  if (c > 0x7fffffffLL || nsplit > 65535 || members > 65535) { set_error("predict: chunk too large for one launch"); return BGP_ERR_INVALID; }
  BGP_TRY(scratch.reserve((size_t)(c * nsplit * members), s));
  predict_var_partial_kernel<<<dim3((unsigned)c, (unsigned)nsplit, (unsigned)members), PV_THREADS, 0, s>>>(
      B, ldb, W, ldw, n, rows, scratch.p, mstride);
  BGP_LAUNCH_CHECK();
  predict_var_finish_kernel<<<dim3((unsigned)std::min<int64_t>((c + 255) / 256, 4 * (int64_t)num_sms()), (unsigned)members),
                              256, 0, s>>>(scratch.p, (int)nsplit, kdiag, c, var, vstride);
  BGP_LAUNCH_CHECK();
  return BGP_OK;
}
int predict_var_launch(const double* B, int64_t ldb, const double* W, int64_t ldw, int64_t n, int64_t c,
                       const double* kdiag, double* var, DevBuf<double>& scratch, cudaStream_t s) {
  return predict_var_batch_launch(B, ldb, W, ldw, n, c, kdiag, var, 1, 0, 0, scratch, s);
}

// C[j*ldc + i] += sum_s slices[s*m*nn + j*m + i], s ascending; `lower`: only i >= j, mirrored to C[i*ldc + j]
// (member blockIdx.y of a batch: slices + y * nsplit * m * nn, C + y * cstride)
__global__ void predict_slices_add_kernel(const double* __restrict__ slices, int nsplit, int64_t m, int64_t nn,
                                          double* __restrict__ C, int64_t ldc, int lower, int64_t cstride) {
  const int64_t total = m * nn;
  slices += blockIdx.y * nsplit * total;
  C += blockIdx.y * cstride;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t j = t / m, i = t - j * m;
    if (lower && i < j) continue;
    double s = 0.0;
    for (int sp = 0; sp < nsplit; ++sp) s += slices[(int64_t)sp * total + t];
    const double v = C[j * ldc + i] + s;
    C[j * ldc + i] = v;
    if (lower && i != j) C[i * ldc + j] = v;
  }
}

// C[i*ldc + j] = C[j*ldc + i] for i > j: the upper triangle of the n x n C from its lower one (member blockIdx.y:
// C + y * cstride)
__global__ void mirror_lower_kernel(double* __restrict__ C, int64_t n, int64_t ldc, int64_t cstride) {
  const int64_t total = n * n;
  C += blockIdx.y * cstride;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t j = t / n, i = t - j * n;
    if (i > j) C[i * ldc + j] = C[j * ldc + i];
  }
}

// The split-K plan of the covariance product (m x nn, K deep): nsplit slices of klen (a multiple of GD_BK) each
void predict_gemm_plan(int64_t m, int64_t nn, int64_t K, int64_t* nsplit_out, int64_t* klen_out) {
  const int64_t tiles = ((m + GD_BM - 1) / GD_BM) * ((nn + GD_BN - 1) / GD_BN);
  int64_t nsplit = (2 * (int64_t)num_sms() + tiles - 1) / tiles;                   // ~2 CTAs per SM
  nsplit = std::min<int64_t>(nsplit, std::max<int64_t>(1, (K + 255) / 256));      // >= 256 of K per split
  nsplit = std::min<int64_t>(nsplit, std::max<int64_t>(1, PREDICT_BUDGET / (m * nn)));
  int64_t klen = (K + nsplit - 1) / nsplit;
  klen = (klen + GD_BK - 1) / GD_BK * GD_BK;
  *nsplit_out = std::max<int64_t>(1, (K + klen - 1) / klen);
  *klen_out = klen;
}

// C (m x nn, column-major ldc) -= A'B' with A'(i, k) = A[i*lda + k], B'(k, j) = B[j*ldb + k], k < K: the (1, 1) DMMA
// variant split over K into nsplit zeroed slices (each one GD_SUB target), then added into C in a fixed order.  With
// one slice the product is subtracted from C directly, with no slice buffer: C - x is the value C + (0 - x) that the
// slice path gives (up to the sign of an exact zero).
// `lower` (m == nn, A == B): only the lower triangle is computed and the result is mirrored, so C stays exactly symmetric.
// `members` > 1: member b uses A and B + b * abstride and C + b * cstride; all members' slices go through one DMMA
// launch (nsplit * members descriptors, member-major) and one add, so the launch count does not depend on members
// while nsplit * members <= 65535.
// `b_kcontig` false (gemm_sub_split_bt): B'(k, j) = B[k*ldb + j] instead, the (1, 0) DMMA variant.
static int gemm_sub_split(const double* A, int64_t lda, const double* B, int64_t ldb, bool b_kcontig, int64_t m,
                          int64_t nn, int64_t K, bool lower, double* C, int64_t ldc, int members, int64_t abstride,
                          int64_t cstride, DevBuf<double>& slices, DevBuf<GemmDesc>& descs, cudaStream_t s) {
  if (m <= 0 || nn <= 0 || members <= 0) return BGP_OK;
  if (m > 0x7fffffffLL || nn > 0x7fffffffLL || K > 0x7fffffffLL) { set_error("predict: GEMM too large"); return BGP_ERR_INVALID; }
  if (members > 65535) { set_error("predict: more than 65535 members in one launch"); return BGP_ERR_INVALID; }
  int64_t nsplit, klen;
  predict_gemm_plan(m, nn, K, &nsplit, &klen);
  const bool direct = nsplit == 1;
  const int64_t slice = m * nn;
  const int64_t nslices = nsplit * members;
  if (!direct) {
    BGP_TRY(slices.reserve((size_t)(slice * nslices), s));
    BGP_CUDA(cudaMemsetAsync(slices.p, 0, sizeof(double) * slice * nslices, s));
  }
  std::vector<GemmDesc> hd((size_t)nslices);
  for (int64_t mb = 0; mb < members; ++mb)
    for (int64_t sp = 0; sp < nsplit; ++sp) {
      const int64_t k0 = sp * klen;
      GemmDesc& d = hd[(size_t)(mb * nsplit + sp)];
      d.A = A + mb * abstride + k0; d.lda = lda;
      d.B = B + mb * abstride + (b_kcontig ? k0 : k0 * ldb); d.ldb = ldb;
      if (direct) { d.C = C + mb * cstride; d.ldc = ldc; }
      else { d.C = slices.p + (mb * nsplit + sp) * slice; d.ldc = m; }
      d.M = (int)m; d.N = (int)nn; d.K = (int)std::max<int64_t>(0, std::min(klen, K - k0));
      d.mode = GD_SUB | (lower ? GD_LOWER : 0);
    }
  BGP_TRY(descs.reserve((size_t)nslices, s));
  BGP_CUDA(cudaMemcpyAsync(descs.p, hd.data(), sizeof(GemmDesc) * nslices, cudaMemcpyHostToDevice, s));
  if (b_kcontig) BGP_TRY((gemm_dmma_launch<true, true>(descs.p, (int)nslices, (int)m, (int)nn, nullptr, s)));
  else BGP_TRY((gemm_dmma_launch<true, false>(descs.p, (int)nslices, (int)m, (int)nn, nullptr, s)));
  if (direct) {
    if (lower) {
      mirror_lower_kernel<<<dim3((unsigned)std::min<int64_t>((slice + 255) / 256, 8 * (int64_t)num_sms()), (unsigned)members),
                            256, 0, s>>>(C, m, ldc, cstride);
      BGP_LAUNCH_CHECK();
    }
    return BGP_OK;
  }
  predict_slices_add_kernel<<<dim3((unsigned)std::min<int64_t>((slice + 255) / 256, 8 * (int64_t)num_sms()), (unsigned)members),
                              256, 0, s>>>(slices.p, (int)nsplit, m, nn, C, ldc, lower ? 1 : 0, cstride);
  BGP_LAUNCH_CHECK();
  return BGP_OK;
}
int predict_gemm_sub_members(const double* A, int64_t lda, const double* B, int64_t ldb, int64_t m, int64_t nn,
                             int64_t K, bool lower, double* C, int64_t ldc, int members, int64_t abstride,
                             int64_t cstride, DevBuf<double>& slices, DevBuf<GemmDesc>& descs, cudaStream_t s) {
  return gemm_sub_split(A, lda, B, ldb, true, m, nn, K, lower, C, ldc, members, abstride, cstride, slices, descs, s);
}
int predict_gemm_sub(const double* A, int64_t lda, const double* B, int64_t ldb, int64_t m, int64_t nn, int64_t K,
                     bool lower, double* C, int64_t ldc, DevBuf<double>& slices, DevBuf<GemmDesc>& descs, cudaStream_t s) {
  return predict_gemm_sub_members(A, lda, B, ldb, m, nn, K, lower, C, ldc, 1, 0, 0, slices, descs, s);
}
// predict_gemm_sub with B'(k, j) = B[k*ldb + j]: C -= A' B^T for a column-major B (n x K), consumed as stored
int predict_gemm_sub_bt_members(const double* A, int64_t lda, const double* B, int64_t ldb, int64_t m, int64_t nn,
                                int64_t K, bool lower, double* C, int64_t ldc, int members, int64_t abstride,
                                int64_t cstride, DevBuf<double>& slices, DevBuf<GemmDesc>& descs, cudaStream_t s) {
  return gemm_sub_split(A, lda, B, ldb, false, m, nn, K, lower, C, ldc, members, abstride, cstride, slices, descs, s);
}
int predict_gemm_sub_bt(const double* A, int64_t lda, const double* B, int64_t ldb, int64_t m, int64_t nn, int64_t K,
                        bool lower, double* C, int64_t ldc, DevBuf<double>& slices, DevBuf<GemmDesc>& descs,
                        cudaStream_t s) {
  return predict_gemm_sub_bt_members(A, lda, B, ldb, m, nn, K, lower, C, ldc, 1, 0, 0, slices, descs, s);
}

}  // namespace bgp

using namespace bgp;

extern "C" {

int bgp_kmat_matvec(const bgp_kernel_spec_t* spec, const double* x1, int64_t n1, const double* x2, int64_t n2,
                    const double* diag, const double* v, int64_t nrhs, double* out) {
  BGP_TRY(require_device());
  DevProgram P;
  BGP_TRY(build_dev_program(spec, &P));
  if (n1 < 0 || n2 < 0 || nrhs < 0) { set_error("negative size"); return BGP_ERR_INVALID; }
  if (diag && n1 != n2) { set_error("dimension mismatch: a diagonal term needs a square operator"); return BGP_ERR_DIM; }
  if (n1 == 0 || nrhs == 0) return BGP_OK;
  cudaStream_t s = 0;
  const int nd = P.ndim;
  const bool same = (x1 == x2 && n1 == n2);
  DevBuf<DevProgram> dprog;
  DevBuf<double> dx1, dx2, dv, dd, dout, scratch;
  BGP_TRY(upload_program(P, dprog, s));
  BGP_TRY(dx1.alloc((size_t)n1 * nd, s));
  BGP_CUDA(cudaMemcpyAsync(dx1.p, x1, sizeof(double) * n1 * nd, cudaMemcpyHostToDevice, s));
  const double* px2 = dx1.p;
  if (!same) {
    BGP_TRY(dx2.alloc((size_t)n2 * nd, s));
    if (n2) BGP_CUDA(cudaMemcpyAsync(dx2.p, x2, sizeof(double) * n2 * nd, cudaMemcpyHostToDevice, s));
    px2 = dx2.p;
  }
  BGP_TRY(dv.alloc((size_t)std::max<int64_t>(n2, 1) * nrhs, s));
  if (n2) BGP_CUDA(cudaMemcpyAsync(dv.p, v, sizeof(double) * n2 * nrhs, cudaMemcpyHostToDevice, s));
  if (diag) {
    BGP_TRY(dd.alloc((size_t)n1, s));
    BGP_CUDA(cudaMemcpyAsync(dd.p, diag, sizeof(double) * n1, cudaMemcpyHostToDevice, s));
  }
  BGP_TRY(dout.alloc((size_t)n1 * nrhs, s));
  BGP_TRY(kmat_matvec_launch(dprog.p, nd, dx1.p, n1, px2, n2, diag ? dd.p : nullptr, dv.p, n2, nrhs, dout.p, n1, scratch, s));
  BGP_CUDA(cudaMemcpyAsync(out, dout.p, sizeof(double) * n1 * nrhs, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  return BGP_OK;
}

int bgp_kmat_matvec_dev(const bgp_kernel_spec_t* spec, const double* x1_dev, int64_t n1, const double* x2_dev, int64_t n2,
                        const double* diag_dev, const double* v_dev, int64_t nrhs, double* out_dev) {
  BGP_TRY(require_device());
  DevProgram P;
  BGP_TRY(build_dev_program(spec, &P));
  if (n1 < 0 || n2 < 0 || nrhs < 0) { set_error("negative size"); return BGP_ERR_INVALID; }
  if (diag_dev && n1 != n2) { set_error("dimension mismatch: a diagonal term needs a square operator"); return BGP_ERR_DIM; }
  DevBuf<DevProgram> dprog;
  DevBuf<double> scratch;
  BGP_TRY(upload_program(P, dprog, 0));
  BGP_TRY(kmat_matvec_launch(dprog.p, P.ndim, x1_dev, n1, x2_dev, n2, diag_dev, v_dev, n2, nrhs, out_dev, n1, scratch, 0));
  BGP_CUDA(cudaStreamSynchronize(0));
  return BGP_OK;
}

static int x1_gradient_matvec_args(const DevProgram& P, int64_t n1, int64_t n2, int64_t ldv) {
  if (n1 < 0 || n2 < 0) { set_error("negative size"); return BGP_ERR_INVALID; }
  if (ldv != 0 && ldv < n2) { set_error("dimension mismatch: ldv %lld is neither 0 nor >= n2 %lld", (long long)ldv, (long long)n2); return BGP_ERR_DIM; }
  if (P.ndim > BGP_MAX_DIM) { set_error("input-coordinate gradients support at most %d dimensions (got %d)", BGP_MAX_DIM, P.ndim); return BGP_ERR_INVALID; }
  return BGP_OK;
}

int bgp_kmat_x1_gradient_matvec(const bgp_kernel_spec_t* spec, const double* x1, int64_t n1, const double* x2,
                                int64_t n2, const double* v, int64_t ldv, double scale, int32_t add_prior, double* out) {
  BGP_TRY(require_device());
  DevProgram P;
  BGP_TRY(build_dev_program(spec, &P));
  BGP_TRY(x1_gradient_matvec_args(P, n1, n2, ldv));
  if (n1 == 0) return BGP_OK;
  cudaStream_t s = 0;
  const int nd = P.ndim;
  const int64_t nv = ldv == 0 ? n2 : ldv * (n1 - 1) + n2;
  DevBuf<DevProgram> dprog;
  DevBuf<double> dx1, dx2, dv, dout, scratch;
  BGP_TRY(upload_program(P, dprog, s));
  BGP_TRY(dx1.alloc((size_t)n1 * nd, s));
  BGP_CUDA(cudaMemcpyAsync(dx1.p, x1, sizeof(double) * n1 * nd, cudaMemcpyHostToDevice, s));
  BGP_TRY(dx2.alloc((size_t)std::max<int64_t>(n2, 1) * nd, s));
  if (n2) BGP_CUDA(cudaMemcpyAsync(dx2.p, x2, sizeof(double) * n2 * nd, cudaMemcpyHostToDevice, s));
  BGP_TRY(dv.alloc((size_t)std::max<int64_t>(nv, 1), s));
  if (nv) BGP_CUDA(cudaMemcpyAsync(dv.p, v, sizeof(double) * nv, cudaMemcpyHostToDevice, s));
  BGP_TRY(dout.alloc((size_t)n1 * nd, s));
  BGP_TRY(kmat_x1_grad_matvec_launch(P, dprog.p, dx1.p, n1, dx2.p, n2, dv.p, ldv, scale, add_prior, dout.p, scratch, s));
  BGP_CUDA(cudaMemcpyAsync(out, dout.p, sizeof(double) * n1 * nd, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  return BGP_OK;
}

int bgp_kmat_x1_gradient_matvec_dev(const bgp_kernel_spec_t* spec, const double* x1_dev, int64_t n1,
                                    const double* x2_dev, int64_t n2, const double* v_dev, int64_t ldv, double scale,
                                    int32_t add_prior, double* out_dev) {
  BGP_TRY(require_device());
  DevProgram P;
  BGP_TRY(build_dev_program(spec, &P));
  BGP_TRY(x1_gradient_matvec_args(P, n1, n2, ldv));
  DevBuf<DevProgram> dprog;
  DevBuf<double> scratch;
  BGP_TRY(upload_program(P, dprog, 0));
  BGP_TRY(kmat_x1_grad_matvec_launch(P, dprog.p, x1_dev, n1, x2_dev, n2, v_dev, ldv, scale, add_prior, out_dev, scratch, 0));
  BGP_CUDA(cudaStreamSynchronize(0));
  return BGP_OK;
}

int bgp_kmat_gradient_contract(const bgp_kernel_spec_t* spec, const uint32_t* which, const double* x, int64_t n,
                               const double* A, double* out) {
  BGP_TRY(require_device());
  DevProgram P;
  BGP_TRY(build_dev_program(spec, &P));
  const int np = P.n_params_total, nd = P.ndim;
  if (n < 0) { set_error("negative size"); return BGP_ERR_INVALID; }
  if (np > 64) { set_error("gradient supports at most 64 hyper-parameters"); return BGP_ERR_INVALID; }
  for (int q = 0; q < np; ++q) out[q] = 0.0;
  if (np == 0 || n == 0) return BGP_OK;
  cudaStream_t s = 0;
  DevBuf<DevProgram> dprog;
  DevBuf<double> dx, dA, dg, scratch;
  DevBuf<unsigned> dw;
  BGP_TRY(upload_program(P, dprog, s));
  BGP_TRY(dx.alloc((size_t)n * nd, s));
  BGP_CUDA(cudaMemcpyAsync(dx.p, x, sizeof(double) * n * nd, cudaMemcpyHostToDevice, s));
  BGP_TRY(dA.alloc((size_t)n * n, s));
  BGP_CUDA(cudaMemcpyAsync(dA.p, A, sizeof(double) * n * n, cudaMemcpyHostToDevice, s));
  BGP_TRY(dw.alloc(np, s));
  BGP_CUDA(cudaMemcpyAsync(dw.p, which, sizeof(unsigned) * np, cudaMemcpyHostToDevice, s));
  BGP_TRY(dg.alloc(np, s));
  BGP_TRY(kmat_grad_contract_launch(dprog.p, nd, np, dw.p, dx.p, n, dA.p, n, nullptr, 0.0, 1.0, dg.p, nullptr, scratch, s));
  BGP_CUDA(cudaMemcpyAsync(out, dg.p, sizeof(double) * np, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  return BGP_OK;
}

}  // extern "C"
