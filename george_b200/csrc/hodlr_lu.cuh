// hodlr_lu.cuh — the Woodbury step of a HODLR level when the 2r x 2r matrix S does not fit one CTA's shared memory
// (r > 71): blocked right-looking LU with partial pivoting, batched over the nodes of the level, trailing updates and
// the multi-right-hand-side triangular solves on DMMA (gemm_dmma.cuh).
//
// Replaces Eigen::FullPivLU of hodlr.h:228-234 (factorize), :90-93 (log-det) and :250 (lu_.solve) for large ranks;
// partial pivoting gives the same determinant / solution up to rounding.
//
//   for each block column k0 (LU_NB wide):
//     lu_panel_kernel   one CTA per node: pivot search, row swap inside the panel, scale, rank-1 updates of the panel
//     lu_swap_kernel    the panel's row interchanges applied to the columns left and right of it
//     lu_trsm_kernel    U12 = L11^-1 S12                       (one thread per column, L11 in shared memory)
//     gemm_dmma         S22 -= L21 U12
//   solve (n x ncols right-hand sides, column-major):
//     lu_laswp_kernel, then per block: lu_trsm_kernel<lower> + gemm_dmma (forward), lu_trsm_kernel<upper> + gemm_dmma
//     (backward).
#pragma once

#include <vector>

#include "gemm_dmma.cuh"

namespace bgp {

constexpr int LU_NB = 32;
constexpr int LU_PANEL_THREADS = 512;
constexpr int LU_TRSM_THREADS = 128;

struct LuNode {
  double* S;       // n x n, column-major, overwritten by L\U
  int* piv;        // n row interchanges (LAPACK convention: row k <-> piv[k], applied in order)
  double* logdet;  // log|det S|
};

struct TrsmDesc {
  const double* T;  // nb x nb triangle (column-major, ldt)
  double* X;        // nb x ncols block it is applied to (column-major, ldx)
  int64_t ldt, ldx;
  int nb, ncols;
};

// (|value| max, lowest index on ties) over the block; result valid in every thread
__device__ __forceinline__ void lu_block_argmax(double& v, int& i, double* red, int* redi) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  warp_argmax(v, i);
  __syncthreads();
  if (lane == 0) { red[w] = v; redi[w] = i; }
  __syncthreads();
  double tv = (lane < nw) ? red[lane] : -1.0;
  int ti = (lane < nw) ? redi[lane] : 0x7fffffff;
  warp_argmax(tv, ti);
  v = tv; i = ti;
}

// S = [[I, W_1[:, own]], [W_0[:, own], I]] from the node's (2r x ncols, ld 2r) Gram block: rows [0, r) hold V1^T X2,
// rows [r, 2r) hold V0^T X1.  grid = (element chunk, node)
__global__ void lu_assemble_kernel(const LuNode* __restrict__ nodes, const double* __restrict__ W, int64_t w_stride_node,
                                   int r, int own_off) {
  const int n = 2 * r;
  const double* Wn = W + (int64_t)blockIdx.y * w_stride_node;
  double* S = nodes[blockIdx.y].S;
  const int64_t total = (int64_t)n * n;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(t % n), j = (int)(t / n);
    double v = (i == j) ? 1.0 : 0.0;
    if (i < r && j >= r) v = Wn[(int64_t)(own_off + j - r) * n + i];
    else if (i >= r && j < r) v = Wn[(int64_t)(own_off + j) * n + i];
    S[t] = v;
  }
}

// unblocked LU of the panel S[k0:n, k0:k0+nb]; one CTA per node
__global__ void __launch_bounds__(LU_PANEL_THREADS) lu_panel_kernel(const LuNode* __restrict__ nodes, int n, int k0, int nb) {
  __shared__ double red[32];
  __shared__ int redi[32];
  __shared__ double srow[LU_NB];
  const LuNode nd = nodes[blockIdx.x];
  double* S = nd.S;
  double ld = 0.0;
  for (int j = 0; j < nb; ++j) {
    const int col = k0 + j;
    double* cj = S + (int64_t)col * n;
    double best = -1.0;
    int bi = 0x7fffffff;
    for (int i = col + threadIdx.x; i < n; i += blockDim.x) {
      const double a = fabs(cj[i]);
      if (a > best) { best = a; bi = i; }
    }
    lu_block_argmax(best, bi, red, redi);
    // nothing comparable below the diagonal (every entry NaN): no interchange, the NaN pivot carries into log|det| and
    // the solve, as small_solve_kernel does.  Without this the sentinel index would be used as a row.
    const int p = bi == 0x7fffffff ? col : bi;
    if (threadIdx.x == 0) nd.piv[col] = p;
    // row interchange inside the panel; stage the new pivot row
    if (threadIdx.x < nb) {
      double* c = S + (int64_t)(k0 + threadIdx.x) * n;
      const double a = c[col], b = c[p];
      if (p != col) { c[col] = b; c[p] = a; }
      srow[threadIdx.x] = b;
    }
    __syncthreads();
    const double dkk = srow[j];
    if (threadIdx.x == 0) ld += log(fabs(dkk));
    const double inv = 1.0 / dkk;
    // scale the column and apply the rank-1 update to the rest of the panel: the row's entries are fetched in batches
    // of 16 explicit global loads (S comes from a descriptor, so plain accesses would serialise on possible aliasing)
    for (int i = col + 1 + threadIdx.x; i < n; i += blockDim.x) {
      const double l = gd_ld_global(cj + i) * inv;
      gd_st_global(cj + i, l);
      double* ri = S + (int64_t)k0 * n + i;  // element (i, k0 + jj) at ri[jj * n]
#pragma unroll
      for (int h0 = 0; h0 < LU_NB; h0 += 16) {
        if (h0 + 15 <= j || h0 >= nb) continue;
        double rv[16];
#pragma unroll
        for (int q = 0; q < 16; ++q) {
          const int jj = h0 + q;
          rv[q] = (jj > j && jj < nb) ? gd_ld_global(ri + (int64_t)jj * n) : 0.0;
        }
#pragma unroll
        for (int q = 0; q < 16; ++q) {
          const int jj = h0 + q;
          if (jj > j && jj < nb) gd_st_global(ri + (int64_t)jj * n, rv[q] - l * srow[jj]);
        }
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *nd.logdet = (k0 == 0 ? 0.0 : *nd.logdet) + ld;
}

// apply the panel's interchanges to the columns outside it.  grid = (column chunk, node)
__global__ void lu_swap_kernel(const LuNode* __restrict__ nodes, int n, int k0, int nb) {
  const LuNode nd = nodes[blockIdx.y];
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n || (c >= k0 && c < k0 + nb)) return;
  double* col = nd.S + (int64_t)c * n;
  for (int j = 0; j < nb; ++j) {
    const int k = k0 + j, p = nd.piv[k];
    if (p != k) { const double a = col[k]; col[k] = col[p]; col[p] = a; }
  }
}

// all n interchanges applied to the rows of the right-hand sides R (n x ncols, ld ldr).  grid = (column chunk, node)
__global__ void lu_laswp_kernel(const LuNode* __restrict__ nodes, int n, double* __restrict__ R, int64_t r_stride_node,
                                int64_t ldr, int ncols) {
  const LuNode nd = nodes[blockIdx.y];
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= ncols) return;
  double* col = R + (int64_t)blockIdx.y * r_stride_node + (int64_t)c * ldr;
  for (int k = 0; k < n; ++k) {
    const int p = nd.piv[k];
    if (p != k) { const double a = col[k]; col[k] = col[p]; col[p] = a; }
  }
}

// X <- T^-1 X for an nb x nb triangle T (unit lower, or upper with its diagonal).  One thread per column of X.
// grid = (column chunk, descriptor)
template <bool UPPER>
__global__ void __launch_bounds__(LU_TRSM_THREADS) lu_trsm_kernel(const TrsmDesc* __restrict__ descs) {
  __shared__ double sT[LU_NB][LU_NB + 1];
  const TrsmDesc d = descs[blockIdx.y];
  if (blockIdx.x * LU_TRSM_THREADS >= d.ncols) return;
  for (int t = threadIdx.x; t < LU_NB * LU_NB; t += LU_TRSM_THREADS) {
    const int i = t % LU_NB, j = t / LU_NB;
    sT[i][j] = (i < d.nb && j < d.nb) ? d.T[(int64_t)j * d.ldt + i] : (i == j ? 1.0 : 0.0);
  }
  __syncthreads();
  const int c = blockIdx.x * LU_TRSM_THREADS + threadIdx.x;
  if (c >= d.ncols) return;
  double* xc = d.X + (int64_t)c * d.ldx;
  double x[LU_NB];
#pragma unroll
  for (int i = 0; i < LU_NB; ++i) x[i] = (i < d.nb) ? xc[i] : 0.0;
  if (!UPPER) {
#pragma unroll
    for (int j = 0; j < LU_NB; ++j) {
#pragma unroll
      for (int i = j + 1; i < LU_NB; ++i) x[i] -= sT[i][j] * x[j];
    }
  } else {
#pragma unroll
    for (int j = LU_NB - 1; j >= 0; --j) {
      x[j] /= sT[j][j];
#pragma unroll
      for (int i = 0; i < j; ++i) x[i] -= sT[i][j] * x[j];
    }
  }
#pragma unroll
  for (int i = 0; i < LU_NB; ++i)
    if (i < d.nb) xc[i] = x[i];
}

// ---- host orchestration ---------------------------------------------------------------------------------------
struct LuWorkspace {
  DevBuf<LuNode> d_nodes;
  DevBuf<TrsmDesc> d_trsm;
  DevBuf<GemmDesc> d_gemm;
};

template <typename T>
static int lu_upload(DevBuf<T>& buf, const std::vector<T>& v, cudaStream_t s) {
  if (v.empty()) return BGP_OK;
  BGP_TRY(buf.reserve(v.size(), s));
  BGP_CUDA(cudaMemcpyAsync(buf.p, v.data(), sizeof(T) * v.size(), cudaMemcpyHostToDevice, s));
  return BGP_OK;
}

// factor every S of the batch (all n x n) in place; pivots, log|det| written through the LuNode pointers
static int lu_factor_batch(LuWorkspace& ws, const std::vector<LuNode>& nodes, int n, cudaStream_t s) {
  const int nn = (int)nodes.size();
  if (nn == 0 || n == 0) return BGP_OK;
  const int nsteps = (n + LU_NB - 1) / LU_NB;
  std::vector<TrsmDesc> td((size_t)nsteps * nn);
  std::vector<GemmDesc> gd((size_t)nsteps * nn);
  for (int t = 0; t < nsteps; ++t) {
    const int k0 = t * LU_NB, nb = std::min(LU_NB, n - k0), rem = n - k0 - nb;
    for (int b = 0; b < nn; ++b) {
      double* S = nodes[b].S;
      TrsmDesc& T = td[(size_t)t * nn + b];
      T.T = S + (int64_t)k0 * n + k0; T.X = S + (int64_t)(k0 + nb) * n + k0; T.ldt = n; T.ldx = n; T.nb = nb; T.ncols = rem;
      GemmDesc& G = gd[(size_t)t * nn + b];
      G.A = S + (int64_t)k0 * n + (k0 + nb); G.B = S + (int64_t)(k0 + nb) * n + k0; G.C = S + (int64_t)(k0 + nb) * n + (k0 + nb);
      G.M = rem; G.N = rem; G.K = nb; G.mode = GD_SUB; G.lda = n; G.ldb = n; G.ldc = n;
    }
  }
  BGP_TRY(lu_upload(ws.d_nodes, nodes, s));
  BGP_TRY(lu_upload(ws.d_trsm, td, s));
  BGP_TRY(lu_upload(ws.d_gemm, gd, s));
  for (int t = 0; t < nsteps; ++t) {
    const int k0 = t * LU_NB, nb = std::min(LU_NB, n - k0), rem = n - k0 - nb;
    lu_panel_kernel<<<nn, LU_PANEL_THREADS, 0, s>>>(ws.d_nodes.p, n, k0, nb);
    BGP_LAUNCH_CHECK();
    if (n > nb) {
      dim3 grid((n + 127) / 128, nn);
      lu_swap_kernel<<<grid, 128, 0, s>>>(ws.d_nodes.p, n, k0, nb);
      BGP_LAUNCH_CHECK();
    }
    if (rem > 0) {
      dim3 grid((rem + LU_TRSM_THREADS - 1) / LU_TRSM_THREADS, nn);
      lu_trsm_kernel<false><<<grid, LU_TRSM_THREADS, 0, s>>>(ws.d_trsm.p + (size_t)t * nn);
      BGP_LAUNCH_CHECK();
      BGP_TRY((gemm_dmma_launch<false, true>(ws.d_gemm.p + (size_t)t * nn, nn, rem, rem, nullptr, s)));
    }
  }
  return BGP_OK;
}

// R_b <- S_b^-1 R_b for every node b: R_b = R + b * r_stride_node, n x ncols, column-major with ld ldr.
// (ws.d_nodes must hold `nodes`: lu_factor_batch uploads it; a solve-only caller passes upload_nodes = true.)
static int lu_solve_batch(LuWorkspace& ws, const std::vector<LuNode>& nodes, int n, double* R, int64_t r_stride_node,
                          int64_t ldr, int ncols, bool upload_nodes, cudaStream_t s) {
  const int nn = (int)nodes.size();
  if (nn == 0 || n == 0 || ncols == 0) return BGP_OK;
  const int nsteps = (n + LU_NB - 1) / LU_NB;
  // descriptors: [forward step t][node] then [backward step t][node]
  std::vector<TrsmDesc> td((size_t)2 * nsteps * nn);
  std::vector<GemmDesc> gd((size_t)2 * nsteps * nn);
  for (int t = 0; t < nsteps; ++t) {
    const int k0 = t * LU_NB, nb = std::min(LU_NB, n - k0), rem = n - k0 - nb;
    for (int b = 0; b < nn; ++b) {
      const double* S = nodes[b].S;
      double* Rb = R + (int64_t)b * r_stride_node;
      TrsmDesc T;
      T.T = S + (int64_t)k0 * n + k0; T.X = Rb + k0; T.ldt = n; T.ldx = ldr; T.nb = nb; T.ncols = ncols;
      td[(size_t)t * nn + b] = T;
      td[(size_t)(nsteps + t) * nn + b] = T;
      GemmDesc F;  // forward: R[k0+nb:n] -= L21 R[k0:k0+nb]
      F.A = S + (int64_t)k0 * n + (k0 + nb); F.B = Rb + k0; F.C = Rb + k0 + nb;
      F.M = rem; F.N = ncols; F.K = nb; F.mode = GD_SUB; F.lda = n; F.ldb = ldr; F.ldc = ldr;
      gd[(size_t)t * nn + b] = F;
      GemmDesc Bk;  // backward: R[0:k0] -= U01 R[k0:k0+nb]
      Bk.A = S + (int64_t)k0 * n; Bk.B = Rb + k0; Bk.C = Rb;
      Bk.M = k0; Bk.N = ncols; Bk.K = nb; Bk.mode = GD_SUB; Bk.lda = n; Bk.ldb = ldr; Bk.ldc = ldr;
      gd[(size_t)(nsteps + t) * nn + b] = Bk;
    }
  }
  if (upload_nodes) BGP_TRY(lu_upload(ws.d_nodes, nodes, s));
  BGP_TRY(lu_upload(ws.d_trsm, td, s));
  BGP_TRY(lu_upload(ws.d_gemm, gd, s));
  {
    dim3 grid((ncols + 127) / 128, nn);
    lu_laswp_kernel<<<grid, 128, 0, s>>>(ws.d_nodes.p, n, R, r_stride_node, ldr, ncols);
    BGP_LAUNCH_CHECK();
  }
  dim3 tgrid((ncols + LU_TRSM_THREADS - 1) / LU_TRSM_THREADS, nn);
  for (int t = 0; t < nsteps; ++t) {
    const int k0 = t * LU_NB, nb = std::min(LU_NB, n - k0), rem = n - k0 - nb;
    lu_trsm_kernel<false><<<tgrid, LU_TRSM_THREADS, 0, s>>>(ws.d_trsm.p + (size_t)t * nn);
    BGP_LAUNCH_CHECK();
    if (rem > 0) BGP_TRY((gemm_dmma_launch<false, true>(ws.d_gemm.p + (size_t)t * nn, nn, rem, ncols, nullptr, s)));
  }
  for (int t = nsteps - 1; t >= 0; --t) {
    const int k0 = t * LU_NB;
    lu_trsm_kernel<true><<<tgrid, LU_TRSM_THREADS, 0, s>>>(ws.d_trsm.p + (size_t)(nsteps + t) * nn);
    BGP_LAUNCH_CHECK();
    if (k0 > 0) BGP_TRY((gemm_dmma_launch<false, true>(ws.d_gemm.p + (size_t)(nsteps + t) * nn, nn, k0, ncols, nullptr, s)));
  }
  return BGP_OK;
}

}  // namespace bgp
