// hodlr_leaf.cuh — K4: leaf build + blocked left-looking LDL^T, one CTA per leaf of up to LF_MAX_LEAF rows.
// Replaces get_exact_matrix + Eigen LDLT (hodlr.h:122-133, 225-227, 87-89).  (A 32-column blocked leaf SOLVE was tried
// and measured slower than leaf_solve_kernel for the 1..160 right-hand sides of this path, so it was dropped.)
//
// The leaf is factorised in 32-column panels, left to right.  A panel (rows k0.., columns k0..k0+31) is built in shared
// memory, brought up to date there and written to global memory once, final:
//   (1) build: the panel's kernel entries on and below the diagonal, evaluated by the whole CTA (the 1-D shapes through
//       ShapeEval, the same arithmetic as the interpreter);
//   (2) update: panel -= L(k0:, 0:k0) D L(k0:k0+32, 0:k0)^T on the tensor pipe (mma.sync.m8n8k4.f64): 16 x 32 output
//       tiles dealt to the 8 warps, both operands read straight from the finished columns in global memory (this CTA
//       wrote them, so they come from L1 / L2), the D scaling applied to the B fragment on the fly, no barrier inside;
//   (3) the 32 x 32 diagonal block: LDL^T by one warp, lane = row, the row in registers and each column of L broadcast
//       by shuffles;
//   (4) the rows below it: L21 = A21 L11^-T D^-1, one row per thread, written to global memory.
// No entry of the leaf is read back and rewritten in global memory.
#pragma once

#include "gemm_dmma.cuh"
#include "hodlr_kernels.cuh"

namespace bgp {

constexpr int LF_THREADS = 256;
constexpr int LF_NB = 32;
constexpr int LF_MAX_LEAF = 768;

__host__ __device__ inline int lf_panel_ld(int max_m) { return ((max_m + 15) / 16) * 16 + 4; }

template <int SHAPE>
__global__ void __launch_bounds__(LF_THREADS, 2) leaf_factor_kernel(const DevProgram* __restrict__ gprog,
                                                                    const double* __restrict__ x,
                                                                    const double* __restrict__ diag,
                                                                    const LeafDesc* __restrict__ leaves,
                                                                    double* __restrict__ Lbuf,
                                                                    double* __restrict__ leaf_logdet, int ldp) {
  // dynamic shared memory: the panel [LF_NB][ldp] (column c, leaf row k0 + i at pn[c * ldp + i]), D of the finished
  // columns [ldp], and for the interpreter the staged program
  extern __shared__ __align__(16) double lf_smem[];
  double* pn = lf_smem;
  double* dall = lf_smem + LF_NB * ldp;
  DevProgram* P = reinterpret_cast<DevProgram*>(lf_smem + (LF_NB + 1) * ldp);
  __shared__ double red[32];
  __shared__ double dinv[LF_NB];
  if constexpr (SHAPE == BGP_SHAPE_GENERIC) stage_program(P, gprog);
  __syncthreads();
  const auto fn = ShapeEval<SHAPE>::make(P, gprog);
  const LeafDesc lf = leaves[blockIdx.x];
  const int m = lf.size, nd = gprog->ndim;
  double* A = Lbuf + lf.off;
  const double* xs = x + (int64_t)lf.start * nd;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  double logdet = 0.0;
  for (int k0 = 0; k0 < m; k0 += LF_NB) {
    const int nb = min(LF_NB, m - k0), rem = m - k0;
    // (1) build
    for (int t = threadIdx.x; t < nb * rem; t += LF_THREADS) {
      const int c = t / rem, i = t - c * rem;
      if (i >= c) {
        double v = fn(xs + (int64_t)(k0 + i) * nd, xs + (int64_t)(k0 + c) * nd);
        if (i == c) v += diag[lf.start + k0 + i];
        pn[c * ldp + i] = v;
      }
    }
    __syncthreads();
    // (2) update from the finished columns 0..k0-1
    if (k0 > 0) {
      const int lr = lane >> 2, lc = lane & 3;
      const int n_tiles = (rem + 15) / 16;
      bool bok[4];
#pragma unroll
      for (int b = 0; b < 4; ++b) bok[b] = b * 8 + lr < nb;
      for (int t = warp; t < n_tiles; t += LF_THREADS / 32) {
        const int r0 = t * 16;
        bool aok[2];
#pragma unroll
        for (int a = 0; a < 2; ++a) aok[a] = r0 + a * 8 + lr < rem;
        double acc[2][4][2];
#pragma unroll
        for (int a = 0; a < 2; ++a)
#pragma unroll
          for (int b = 0; b < 4; ++b) { acc[a][b][0] = 0.0; acc[a][b][1] = 0.0; }
#pragma unroll 4
        for (int q0 = 0; q0 < k0; q0 += 4) {
          const int q = q0 + lc;
          const double* Lq = A + (int64_t)q * m + k0;
          const double dq = dall[q];
          double af[2], bf[4];
#pragma unroll
          for (int a = 0; a < 2; ++a) af[a] = aok[a] ? Lq[r0 + a * 8 + lr] : 0.0;
#pragma unroll
          for (int b = 0; b < 4; ++b) bf[b] = bok[b] ? Lq[b * 8 + lr] * dq : 0.0;
#pragma unroll
          for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b) dmma884(acc[a][b][0], acc[a][b][1], af[a], bf[b]);
        }
#pragma unroll
        for (int a = 0; a < 2; ++a) {
          const int i = r0 + a * 8 + lr;
#pragma unroll
          for (int b = 0; b < 4; ++b)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int c = b * 8 + 2 * lc + e;
              if (i < rem && c < nb && i >= c) pn[c * ldp + i] -= acc[a][b][e];
            }
        }
      }
      __syncthreads();
    }
    // (3) warp 0: LDL^T of the diagonal block, lane = row
    if (warp == 0) {
      double w[LF_NB];
#pragma unroll
      for (int j = 0; j < LF_NB; ++j) w[j] = (j <= lane && lane < nb) ? pn[j * ldp + lane] : 0.0;
#pragma unroll
      for (int k = 0; k < LF_NB; ++k) {
        if (k < nb) {
          const double d = __shfl_sync(0xffffffffu, w[k], k);
          const double l = (lane > k && lane < nb) ? w[k] / d : 0.0;
          if (lane > k) w[k] = l;
          const double ld = l * d;
#pragma unroll
          for (int j = k + 1; j < LF_NB; ++j) {
            const double lj = __shfl_sync(0xffffffffu, l, j);
            if (j <= lane) w[j] -= ld * lj;
          }
        }
      }
      if (lane < nb) {
        double* col = A + (int64_t)k0 * m + k0 + lane;  // row k0 + lane of the leaf
        double d = 0.0;
#pragma unroll
        for (int j = 0; j < LF_NB; ++j) {
          if (j < lane) { pn[j * ldp + lane] = w[j]; col[(int64_t)j * m] = w[j]; }
          if (j == lane) d = w[j];
        }
        col[(int64_t)lane * m] = d;
        dall[k0 + lane] = d;
        dinv[lane] = 1.0 / d;
        logdet += log(fabs(d));
      }
    }
    __syncthreads();
    // (4) the rows below the diagonal block (there are some only when the panel is full: nb == LF_NB)
    const volatile double* l11 = pn;  // (volatile: read where used, not hoisted out of the row loop into 528 registers)
    for (int i = LF_NB + threadIdx.x; i < rem; i += LF_THREADS) {
      double w[LF_NB];
#pragma unroll
      for (int j = 0; j < LF_NB; ++j) w[j] = pn[j * ldp + i];
#pragma unroll
      for (int j = 0; j < LF_NB; ++j) {
        double s = w[j];
#pragma unroll
        for (int q = 0; q < j; ++q) s -= w[q] * l11[q * ldp + j];
        w[j] = s;
      }
      double* row = A + (int64_t)k0 * m + k0 + i;
#pragma unroll
      for (int j = 0; j < LF_NB; ++j) row[(int64_t)j * m] = w[j] * dinv[j];
    }
    __syncthreads();
  }
  logdet = block_sum(logdet, red);
  if (threadIdx.x == 0) leaf_logdet[blockIdx.x] = logdet;
}

// dynamic shared memory of leaf_factor_kernel<SHAPE> for leaves of up to max_m rows
__host__ inline size_t lf_smem_bytes(int shape, int max_m) {
  return sizeof(double) * (size_t)(LF_NB + 1) * lf_panel_ld(max_m) + (shape == BGP_SHAPE_GENERIC ? sizeof(DevProgram) : 0);
}

template <int SHAPE>
inline void leaf_factor_launch_shape(int n_leaves, int max_m, cudaStream_t s, const DevProgram* prog, const double* x,
                                     const double* diag, const LeafDesc* leaves, double* L, double* leaf_logdet) {
  const size_t smem = lf_smem_bytes(SHAPE, max_m);
  // (the attribute is per device / context: set it on every call, it is cheap)
  cudaFuncSetAttribute(leaf_factor_kernel<SHAPE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  leaf_factor_kernel<SHAPE><<<n_leaves, LF_THREADS, smem, s>>>(prog, x, diag, leaves, L, leaf_logdet, lf_panel_ld(max_m));
}

// one CTA per leaf; every leaf has at most LF_MAX_LEAF rows
inline void leaf_factor_launch(int shape, int n_leaves, int max_m, cudaStream_t s, const DevProgram* prog,
                               const double* x, const double* diag, const LeafDesc* leaves, double* L,
                               double* leaf_logdet) {
  BGP_SHAPE_SWITCH(shape, (leaf_factor_launch_shape<SHAPE>(n_leaves, max_m, s, prog, x, diag, leaves, L, leaf_logdet)));
}

}  // namespace bgp
