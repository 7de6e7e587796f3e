// hodlr_leaf.cuh — K4: leaf build + blocked left-looking LDL^T, one CTA per leaf of up to LF_MAX_LEAF rows.
// Replaces get_exact_matrix + Eigen LDLT (hodlr.h:122-133, 225-227, 87-89).  (A 32-column blocked leaf SOLVE was tried
// and measured slower than leaf_solve_kernel for the 1..160 right-hand sides of this path, so it was dropped.)
//
// The leaf is factorised in 32-column panels, left to right.  A panel (rows k0.., columns k0..k0+31) is brought up to
// date in shared memory and written to global memory once, final:
//   (1) build: the panel's kernel entries on and below the diagonal, LF_BUILD_ILP independent entries per thread in
//       flight (the 1-D shapes through ShapeEval, the same arithmetic as the interpreter), parked in the panel's own
//       slots of the factor (the diagonal in shared memory) until its turn;
//   (2) update: panel -= L(k0:, 0:k0) D L(k0:k0+32, 0:k0)^T on the tensor pipe (mma.sync.m8n8k4.f64) in 16 x 32 output
//       tiles, both operands read straight from the finished columns in global memory (this CTA wrote them, so they
//       come from L1 / L2), the D scaling applied to the B fragment on the fly;
//   (3) the 32 x 32 diagonal block: right-looking LDL^T by one warp in shared memory, lane = row, with a rolled loop
//       (a fully unrolled register version is ~7k instructions run once per panel by one warp: it streamed through the
//       instruction cache and cost more than the rest of the panel).  The same warp eliminates the identity alongside,
//       which leaves W = L11^-T D^-1 in shared memory;
//   (4) the rows below it: L21 = A21 W on the tensor pipe, 16 x 32 tiles dealt to the 8 warps, written to global memory
//       from the accumulators.
// Warps 1..7 look one panel ahead: while warp 0 runs (3) for panel p they build panel p + 1 and accumulate its update
// over the columns before panel p, none of which depends on panel p.  The accumulators are parked unsubtracted; at
// panel p + 1's turn all warps continue them with panel p's 32 columns and subtract once, so each entry sums its terms
// in the order of a single pass and the factor is bit for bit that of the panel-by-panel schedule (DESIGN.md §6).
#pragma once

#include "gemm_dmma.cuh"
#include "hodlr_kernels.cuh"

namespace bgp {

constexpr int LF_THREADS = 256;
constexpr int LF_NB = 32;
constexpr int LF_MAX_LEAF = 768;
constexpr int LF_LDW = 40;  // leading dimension of W: the B fragments of phase (4) read it without bank conflicts

// panel leading dimension: = 8 (mod 16) doubles, so that the A fragments (4 columns x 8 rows) fill two bank wavefronts
__host__ __device__ inline int lf_panel_ld(int max_m) { return ((max_m + 15) / 16) * 16 + 8; }

// dst[j * ds] -= f * src[j * ss] for j in [lo, hi]: 8 shared-memory loads issued before their stores (one at a time,
// each load would wait for the store before it, which the compiler cannot tell apart from an alias)
__device__ __forceinline__ void lf_axpy(double* dst, int ds, const double* src, int ss, int lo, int hi, double f) {
  for (int j0 = lo; j0 <= hi; j0 += 8) {
    double a[8], b[8];
#pragma unroll
    for (int u = 0; u < 8; ++u)
      if (j0 + u <= hi) { a[u] = dst[(j0 + u) * ds]; b[u] = src[(j0 + u) * ss]; }
#pragma unroll
    for (int u = 0; u < 8; ++u)
      if (j0 + u <= hi) dst[(j0 + u) * ds] = a[u] - f * b[u];
  }
}

template <int SHAPE>
__global__ void __launch_bounds__(LF_THREADS, 2) leaf_factor_kernel(const DevProgram* __restrict__ gprog,
                                                                    const double* __restrict__ x,
                                                                    const double* __restrict__ diag,
                                                                    const LeafDesc* __restrict__ leaves,
                                                                    double* __restrict__ Lbuf,
                                                                    double* __restrict__ leaf_logdet, int ldp) {
  // dynamic shared memory: the panel [LF_NB][ldp] (column c, leaf row k0 + i at pn[c * ldp + i]), D of the finished
  // columns [ldp], W = L11^-T D^-1 of the current panel [LF_NB][LF_LDW] (W(q, n) at w11[q * LF_LDW + n]), and for the
  // interpreter the staged program
  extern __shared__ __align__(16) double lf_smem[];
  double* pn = lf_smem;
  double* dall = lf_smem + LF_NB * ldp;
  double* w11 = dall + ldp;
  DevProgram* P = reinterpret_cast<DevProgram*>(w11 + LF_NB * LF_LDW);
  __shared__ double red[32];
  __shared__ double draw[LF_NB];  // the diagonal kernel entries (+ diag) of the next panel
  if constexpr (SHAPE == BGP_SHAPE_GENERIC) stage_program(P, gprog);
  __syncthreads();
  const auto fn = ShapeEval<SHAPE>::make(P, gprog);
  const LeafDesc lf = leaves[blockIdx.x];
  const int m = lf.size, nd = gprog->ndim;
  double* A = Lbuf + lf.off;
  const double* xs = x + (int64_t)lf.start * nd;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int lr = lane >> 2, lc = lane & 3;  // mma.m8n8k4 fragment coordinates

  // independent kernel evaluations per thread in flight in the build (the interpreter keeps one: its stack is large)
  constexpr int LF_BUILD_ILP = SHAPE == BGP_SHAPE_GENERIC ? 1 : 4;
  // (1) build of the panel at leaf row kp by threads t_first.. (nthreads of them): its kernel entries on and below the
  // diagonal, parked until the panel's turn: off the diagonal in their own slots of the factor, the diagonal in draw
  auto build = [&](int kp, int t_first, int nthreads) {
    const int nb = min(LF_NB, m - kp), rem = m - kp;
    for (int t0 = t_first; t0 < nb * rem; t0 += LF_BUILD_ILP * nthreads) {
      double v[LF_BUILD_ILP];
#pragma unroll
      for (int u = 0; u < LF_BUILD_ILP; ++u) {
        const int t = t0 + u * nthreads, c = t / rem, i = t - c * rem;
        v[u] = (t < nb * rem && i >= c) ? fn(xs + (int64_t)(kp + i) * nd, xs + (int64_t)(kp + c) * nd) : 0.0;
      }
#pragma unroll
      for (int u = 0; u < LF_BUILD_ILP; ++u) {
        const int t = t0 + u * nthreads, c = t / rem, i = t - c * rem;
        if (t < nb * rem && i > c) A[(int64_t)(kp + c) * m + kp + i] = v[u];
        if (t < nb * rem && i == c) draw[c] = v[u] + diag[lf.start + kp + i];
      }
    }
  };
  // (2) update: acc += L(kp + r0.., q) D(q) L(kp + 0..31, q)^T over the finished columns q in [q_lo, q_hi), a 16 x 32
  // tile of the panel at leaf row kp on the tensor pipe (mma.sync.m8n8k4.f64), both operands read straight from the
  // finished columns in global memory (this CTA wrote them, so they come from L1 / L2), the D scaling applied to the
  // B fragment on the fly
  auto update = [&](double (&acc)[2][4][2], int kp, int r0, int q_lo, int q_hi) {
    const int nb = min(LF_NB, m - kp), rem = m - kp;
    bool aok[2], bok[4];
#pragma unroll
    for (int a = 0; a < 2; ++a) aok[a] = r0 + a * 8 + lr < rem;
#pragma unroll
    for (int b = 0; b < 4; ++b) bok[b] = b * 8 + lr < nb;
#pragma unroll 4
    for (int q0 = q_lo; q0 < q_hi; q0 += 4) {
      const int q = q0 + lc;
      const double* Lq = A + (int64_t)q * m + kp;
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
  };
  // a panel's update accumulators are parked unsubtracted in rows 0..31 of columns 32.. of the leaf, in its strict
  // upper triangle, which no consumer of the factor reads: element f = 8 a + 2 b + e of lane `lane` of tile t at row
  // `lane` of column 32 + 16 t + f, so that a warp stores and loads 256 contiguous bytes.  Only panels from row 64 on
  // park, so their tiles end at column m - 18 or before.
  auto parked = [&](int t, int a, int b, int e) -> double& {
    return A[(int64_t)(LF_NB + 16 * t + 8 * a + 2 * b + e) * m + lane];
  };

  double logdet = 0.0;
  build(0, threadIdx.x, LF_THREADS);
  __syncthreads();
  for (int k0 = 0; k0 < m; k0 += LF_NB) {
    const int nb = min(LF_NB, m - k0), rem = m - k0, k1 = k0 + LF_NB;
    // (2) into shared memory: the panel's kernel entries minus its update, the parked accumulators of the columns
    // before the previous panel continued with the previous panel's 32 columns, so that every entry sums its terms in
    // the order of one pass over the columns 0..k0-1
    for (int t = warp; t < (rem + 15) / 16; t += LF_THREADS / 32) {
      const int r0 = t * 16;
      double acc[2][4][2];
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b)
#pragma unroll
          for (int e = 0; e < 2; ++e) acc[a][b][e] = k0 > LF_NB ? parked(t, a, b, e) : 0.0;
      update(acc, k0, r0, max(k0 - LF_NB, 0), k0);
      // all loads of the kernel entries before the first store (a shared-memory store would hold back the loads after
      // it: the compiler cannot tell pn from draw)
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int i = r0 + a * 8 + lr, c = b * 8 + 2 * lc + e;
            if (i < rem && c < nb && i >= c)
              acc[a][b][e] = (i == c ? draw[c] : A[(int64_t)(k0 + c) * m + k0 + i]) - acc[a][b][e];
          }
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int i = r0 + a * 8 + lr, c = b * 8 + 2 * lc + e;
            if (i < rem && c < nb && i >= c) pn[c * ldp + i] = acc[a][b][e];
          }
    }
    __syncthreads();
    // (3) warp 0: LDL^T of the diagonal block, lane = row i, and T = L11^-1 (starting from the identity, row i of T
    // takes the same eliminations as row i of the block); then W = T^T D^-1.  Meanwhile warps 1..7 look one panel
    // ahead: they build the next panel and accumulate its update from the columns before this one, none of which
    // depends on this panel.
    if (warp == 0) {
      double* t11 = w11;  // T(i, j) at t11[j * LF_LDW + i]
      for (int j = 0; j < LF_NB; ++j) t11[j * LF_LDW + lane] = (j == lane) ? 1.0 : 0.0;
      __syncwarp();
      for (int k = 0; k < nb; ++k) {
        const double d = pn[k * ldp + k];
        const bool below = lane > k && lane < nb;
        const double l = below ? pn[k * ldp + lane] / d : 0.0;
        if (below) pn[k * ldp + lane] = l;
        __syncwarp();
        if (below) {
          const double ld = l * d;
          lf_axpy(pn + lane, ldp, pn + k * ldp, 1, k + 1, lane, ld);
          lf_axpy(t11 + lane, LF_LDW, t11 + k, LF_LDW, 0, k, l);
        }
        __syncwarp();
      }
      if (lane < nb) {
        const double d = pn[lane * ldp + lane];
        const double dinv = 1.0 / d;
        double* col = A + (int64_t)k0 * m + k0 + lane;  // row k0 + lane of the leaf
        for (int j = 0; j < lane; ++j) col[(int64_t)j * m] = pn[j * ldp + lane];
        col[(int64_t)lane * m] = d;
        dall[k0 + lane] = d;
        logdet += log(fabs(d));
        for (int j = 0; j <= lane; ++j) t11[j * LF_LDW + lane] *= dinv;
      }
    } else if (k1 < m) {
      build(k1, threadIdx.x - 32, LF_THREADS - 32);
      if (k0 > 0) {
        for (int t = warp - 1; t < (m - k1 + 15) / 16; t += LF_THREADS / 32 - 1) {
          const int r0 = t * 16;
          double acc[2][4][2];
#pragma unroll
          for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b) { acc[a][b][0] = 0.0; acc[a][b][1] = 0.0; }
          update(acc, k1, r0, 0, k0);
#pragma unroll
          for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b)
#pragma unroll
              for (int e = 0; e < 2; ++e) parked(t, a, b, e) = acc[a][b][e];
        }
      }
    }
    __syncthreads();
    // (4) the rows below the diagonal block (there are some only when the panel is full: nb == LF_NB)
    if (rem > LF_NB) {
      const int n_tiles = (rem - LF_NB + 15) / 16;
      for (int t = warp; t < n_tiles; t += LF_THREADS / 32) {
        const int r0 = LF_NB + t * 16;
        bool aok[2];
#pragma unroll
        for (int a = 0; a < 2; ++a) aok[a] = r0 + a * 8 + lr < rem;
        double acc[2][4][2];
#pragma unroll
        for (int a = 0; a < 2; ++a)
#pragma unroll
          for (int b = 0; b < 4; ++b) { acc[a][b][0] = 0.0; acc[a][b][1] = 0.0; }
#pragma unroll
        for (int q0 = 0; q0 < LF_NB; q0 += 4) {
          const int q = q0 + lc;
          double af[2], bf[4];
#pragma unroll
          for (int a = 0; a < 2; ++a) af[a] = aok[a] ? pn[q * ldp + r0 + a * 8 + lr] : 0.0;
#pragma unroll
          for (int b = 0; b < 4; ++b) bf[b] = w11[q * LF_LDW + b * 8 + lr];
#pragma unroll
          for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b) dmma884(acc[a][b][0], acc[a][b][1], af[a], bf[b]);
        }
#pragma unroll
        for (int a = 0; a < 2; ++a) {
          const int i = r0 + a * 8 + lr;
          if (i < rem) {
#pragma unroll
            for (int b = 0; b < 4; ++b)
#pragma unroll
              for (int e = 0; e < 2; ++e) A[(int64_t)(k0 + b * 8 + 2 * lc + e) * m + k0 + i] = acc[a][b][e];
          }
        }
      }
    }
    __syncthreads();
  }
  logdet = block_sum(logdet, red);
  if (threadIdx.x == 0) leaf_logdet[blockIdx.x] = logdet;
}

// dynamic shared memory of leaf_factor_kernel<SHAPE> for leaves of up to max_m rows
__host__ inline size_t lf_smem_bytes(int shape, int max_m) {
  return sizeof(double) * ((size_t)(LF_NB + 1) * lf_panel_ld(max_m) + LF_NB * LF_LDW) +
         (shape == BGP_SHAPE_GENERIC ? sizeof(DevProgram) : 0);
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
