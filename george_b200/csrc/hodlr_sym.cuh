// hodlr_sym.cuh — device kernels of the HODLR symmetric factor K~ = W W^T (hodlr_sym.cu; Ambikasaran, O'Neil & Singh,
// "Fast symmetric factorization of hierarchical matrices with applications", arXiv:1405.0223).
//
//   W = W_leaf W_{k-1} ... W_0,   W_leaf = blockdiag(L D^1/2) over the leaves,
//   W_l = blockdiag over the nodes v of level l of (I + Q_v X_v Q_v^T),   Q_v = blockdiag(Q_0, Q_1) (orthonormal),
//   W_l^-1 = ... (I + Q_v Y_v Q_v^T).
// Every product sums its terms in a fixed order and no kernel adds floating-point values with atomics, so the factor
// and every application of it are reproducible bit for bit.
#pragma once

#include "common.cuh"

namespace bgp {

// one internal node, listed level by level (deepest level last) in the order of the level's nodes
struct SymNode {
  int start, size, half, rank;  // rank: the node's own ACA rank; columns [rank, r) of its level are zero padding
  int r, ucol;                  // the level's common rank and its first column in the factor panel P
  int64_t x_off;                // X_v at x_off, Y_v at x_off + (2r)^2 (column-major, leading dimension 2r)
  int64_t q_off;                // R_0, R_1, R^-1_0, R^-1_1, G_0, G_1 (r x r each, leading dimension r)
};
struct SymLeaf {
  int start, size, ncols, _pad;  // ncols: ancestor columns of P over the leaf's rows
  int64_t off;                   // the leaf's L D L^T block in the leaf-factor buffer (m x m, column-major)
};

constexpr int SY_THREADS = 256;
constexpr int SY_TN_ROWS = 64;     // rows per shared-memory slab of sym_tn_kernel
constexpr int SY_TN_TQ = 32;       // Q columns per pass
constexpr int SY_TN_TC = 32;       // target columns per CTA
constexpr int SY_TN_CHUNK = 2048;  // rows per CTA: one partial product per chunk, summed in chunk order
constexpr int SY_NN_ROWS = 32;     // rows per CTA of sym_nn_kernel (staged with all of the node's Q columns); fewer,
                                   // down to 1, where r is too large for 32 rows of it in shared memory
constexpr int SY_LEAF_COLS = 8;    // right-hand sides per CTA of the leaf kernels

// ---- leaves ------------------------------------------------------------------------------------------------------

// Positive definiteness of the leaves' D and their log-determinant, one CTA per leaf.  bad_row gets the smallest
// global row whose pivot is not a finite positive number (integer atomics only).
__global__ void __launch_bounds__(SY_THREADS) sym_leaf_check_kernel(const SymLeaf* __restrict__ leaves,
                                                                    const double* __restrict__ Lbuf,
                                                                    double* __restrict__ leaf_logdet,
                                                                    int* __restrict__ bad_row) {
  __shared__ double red[32];
  const SymLeaf lf = leaves[blockIdx.x];
  const double* A = Lbuf + lf.off;
  double s = 0.0;
  for (int i = threadIdx.x; i < lf.size; i += SY_THREADS) {
    const double d = A[(int64_t)i * lf.size + i];
    if (!(d > 0.0) || !isfinite(d)) atomicMin(bad_row, lf.start + i);
    else s += log(d);
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) leaf_logdet[blockIdx.x] = s;
}

// X <- D^-1/2 L^-1 X on each leaf's rows for its `ncols` ancestor columns.  One CTA per (leaf, group of COLS columns),
// the group staged in shared memory; one step per column of L, its rows below the diagonal spread over the threads.
template <int COLS>
__global__ void __launch_bounds__(SY_THREADS) sym_leaf_forward_kernel(const SymLeaf* __restrict__ leaves,
                                                                      const double* __restrict__ Lbuf,
                                                                      double* __restrict__ X, int64_t ldx, int max_m,
                                                                      int ngroups) {
  extern __shared__ double xs[];  // max_m x COLS, column-major
  const SymLeaf lf = leaves[blockIdx.x / ngroups];
  const int c0 = (blockIdx.x % ngroups) * COLS;
  if (c0 >= lf.ncols) return;
  const int nc = min(COLS, lf.ncols - c0), m = lf.size;
  const double* A = Lbuf + lf.off;
  for (int t = threadIdx.x; t < m * COLS; t += SY_THREADS) {
    const int i = t % m, c = t / m;
    xs[c * max_m + i] = c < nc ? X[(int64_t)(c0 + c) * ldx + lf.start + i] : 0.0;
  }
  __syncthreads();
  for (int k = 0; k + 1 < m; ++k) {
    double yk[COLS];
#pragma unroll
    for (int c = 0; c < COLS; ++c) yk[c] = xs[c * max_m + k];
    for (int i = k + 1 + threadIdx.x; i < m; i += SY_THREADS) {
      const double l = A[(int64_t)k * m + i];
#pragma unroll
      for (int c = 0; c < COLS; ++c) xs[c * max_m + i] -= l * yk[c];
    }
    __syncthreads();
  }
  for (int t = threadIdx.x; t < m * nc; t += SY_THREADS) {
    const int i = t % m, c = t / m;
    X[(int64_t)(c0 + c) * ldx + lf.start + i] = xs[c * max_m + i] / sqrt(A[(int64_t)i * m + i]);
  }
}

// Z <- L D^1/2 Z (transpose = 0) or D^1/2 L^T Z (transpose = 1) on every leaf: products, so every row is independent
// once the group is staged.  Non-transposed: a thread per row reads row i of L along its columns (coalesced over the
// threads); transposed: a warp per row reads column i of L (contiguous) and adds its lanes with a fixed butterfly.
template <int COLS>
__global__ void __launch_bounds__(SY_THREADS) sym_leaf_product_kernel(const SymLeaf* __restrict__ leaves,
                                                                      const double* __restrict__ Lbuf,
                                                                      double* __restrict__ Z, int64_t ldz, int ncols,
                                                                      int max_m, int ngroups, int transpose) {
  extern __shared__ double zs[];  // max_m x COLS
  const SymLeaf lf = leaves[blockIdx.x / ngroups];
  const int c0 = (blockIdx.x % ngroups) * COLS;
  if (c0 >= ncols) return;
  const int nc = min(COLS, ncols - c0), m = lf.size;
  const double* A = Lbuf + lf.off;
  for (int t = threadIdx.x; t < m * COLS; t += SY_THREADS) {
    const int i = t % m, c = t / m;
    const double z = c < nc ? Z[(int64_t)(c0 + c) * ldz + lf.start + i] : 0.0;
    zs[c * max_m + i] = transpose ? z : z * sqrt(A[(int64_t)i * m + i]);
  }
  __syncthreads();
  if (!transpose) {
    for (int i = threadIdx.x; i < m; i += SY_THREADS) {
      double acc[COLS];
#pragma unroll
      for (int c = 0; c < COLS; ++c) acc[c] = zs[c * max_m + i];
      for (int k = 0; k < i; ++k) {
        const double l = A[(int64_t)k * m + i];
#pragma unroll
        for (int c = 0; c < COLS; ++c) acc[c] += l * zs[c * max_m + k];
      }
#pragma unroll
      for (int c = 0; c < COLS; ++c)
        if (c < nc) Z[(int64_t)(c0 + c) * ldz + lf.start + i] = acc[c];
    }
  } else {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = warp; i < m; i += SY_THREADS / 32) {
      const double* col = A + (int64_t)i * m;  // L(k, i), k > i
      double acc[COLS];
#pragma unroll
      for (int c = 0; c < COLS; ++c) acc[c] = 0.0;
      for (int k = i + 1 + lane; k < m; k += 32) {
        const double l = col[k];
#pragma unroll
        for (int c = 0; c < COLS; ++c) acc[c] += l * zs[c * max_m + k];
      }
#pragma unroll
      for (int c = 0; c < COLS; ++c) acc[c] = warp_sum(acc[c]);
      if (lane == 0) {
        const double sd = sqrt(col[i]);
#pragma unroll
        for (int c = 0; c < COLS; ++c)
          if (c < nc) Z[(int64_t)(c0 + c) * ldz + lf.start + i] = sd * (zs[c * max_m + i] + acc[c]);
      }
    }
  }
}

// ---- levels ------------------------------------------------------------------------------------------------------

// P[:, ucol + k] = V[:, vcol + k] on the node's rows for its own columns k < rank, zero for the padding k < r.
__global__ void __launch_bounds__(SY_THREADS) sym_copy_kernel(const SymNode* __restrict__ nodes,
                                                              const double* __restrict__ V, int64_t ldv, int vcol,
                                                              double* __restrict__ P, int64_t ldp) {
  const SymNode nd = nodes[blockIdx.y];
  const int i = blockIdx.x * SY_THREADS + threadIdx.x;
  if (i >= nd.size) return;
  for (int k = 0; k < nd.r; ++k)
    P[(int64_t)(nd.ucol + k) * ldp + nd.start + i] = k < nd.rank ? V[(int64_t)(vcol + k) * ldv + nd.start + i] : 0.0;
}

// Partial products  Q_h^T B_h  over one chunk of SY_TN_CHUNK rows of half h of a node: Q_h = the node's own columns of
// P on the half's rows, B_h = columns [bcol0, bcol0 + ncols) of B on the same rows.  Block (node b, half h, chunk k)
// of `part` holds the r x ncols partial (leading dimension r) at ((b * 2 + h) * nchunks + k) * r * ncols.
// grid = (chunk, (node - b0) * 2 + h, column tile): a launch covers the nodes [b0, b0 + gridDim.y / 2) of the level
__global__ void __launch_bounds__(SY_THREADS) sym_tn_kernel(const SymNode* __restrict__ nodes,
                                                            const double* __restrict__ P, int64_t ldp,
                                                            const double* __restrict__ B, int64_t ldb, int bcol0,
                                                            int ncols, double* __restrict__ part, int nchunks, int b0) {
  __shared__ double sq[SY_TN_ROWS][SY_TN_TQ + 1];
  __shared__ double sb[SY_TN_ROWS][SY_TN_TC + 1];
  const SymNode nd = nodes[b0 + (blockIdx.y >> 1)];
  const int h = blockIdx.y & 1;
  const int rs = nd.start + (h ? nd.half : 0), nh = h ? nd.size - nd.half : nd.half;
  const int row_lo = blockIdx.x * SY_TN_CHUNK;
  if (row_lo >= nh || nd.rank == 0) return;
  const int row_hi = min(nh, row_lo + SY_TN_CHUNK);
  const int c0 = blockIdx.z * SY_TN_TC;
  if (c0 >= ncols) return;
  const int nc = min(SY_TN_TC, ncols - c0);
  double* out = part + ((int64_t)(2 * b0 + blockIdx.y) * nchunks + blockIdx.x) * nd.r * ncols;
  const int tq = threadIdx.x & 31, tc = threadIdx.x >> 5;
  for (int q0 = 0; q0 < nd.rank; q0 += SY_TN_TQ) {
    const int nq = min(SY_TN_TQ, nd.rank - q0);
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    for (int i0 = row_lo; i0 < row_hi; i0 += SY_TN_ROWS) {
      const int ni = min(SY_TN_ROWS, row_hi - i0);
      __syncthreads();
      for (int t = threadIdx.x; t < SY_TN_ROWS * SY_TN_TQ; t += SY_THREADS) {
        const int i = t % SY_TN_ROWS, q = t / SY_TN_ROWS;
        sq[i][q] = (i < ni && q < nq) ? P[(int64_t)(nd.ucol + q0 + q) * ldp + rs + i0 + i] : 0.0;
      }
      for (int t = threadIdx.x; t < SY_TN_ROWS * SY_TN_TC; t += SY_THREADS) {
        const int i = t % SY_TN_ROWS, c = t / SY_TN_ROWS;
        sb[i][c] = (i < ni && c < nc) ? B[(int64_t)(bcol0 + c0 + c) * ldb + rs + i0 + i] : 0.0;
      }
      __syncthreads();
#pragma unroll 8
      for (int i = 0; i < SY_TN_ROWS; ++i) {
        const double a = sq[i][tq];
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[e] += a * sb[i][tc + 8 * e];
      }
    }
    if (tq < nq) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int c = tc + 8 * e;
        if (c < nc) out[(int64_t)(c0 + c) * nd.r + q0 + tq] = acc[e];
      }
    }
  }
}

// the sum over the chunks of half h (in chunk order) of entry (q, c) of sym_tn_kernel's partials
__device__ __forceinline__ double sym_chunk_sum(const double* part, int b, int h, int nchunks, int nh, int r, int ncols,
                                                int q, int c) {
  const int nk = (nh + SY_TN_CHUNK - 1) / SY_TN_CHUNK;
  const double* p = part + ((int64_t)(b * 2 + h) * nchunks) * r * ncols + (int64_t)c * r + q;
  double s = 0.0;
  for (int k = 0; k < nk; ++k) s += p[(int64_t)k * r * ncols];
  return s;
}

// In-place lower Cholesky A = L L^T of the leading n x n block (leading dimension ld) by one CTA; the strict upper
// triangle is not read.  Returns 0, or k + 1 when pivot k is not a finite positive number (the same on every thread).
__device__ int cta_cholesky(double* A, int n, int ld) {
  for (int k = 0; k < n; ++k) {
    const double piv = A[(int64_t)k * ld + k];
    if (!(piv > 0.0) || !isfinite(piv)) return k + 1;
    const double lkk = sqrt(piv);
    __syncthreads();  // every thread has read the pivot
    for (int i = k + threadIdx.x; i < n; i += blockDim.x) A[(int64_t)k * ld + i] = i == k ? lkk : A[(int64_t)k * ld + i] / lkk;
    __syncthreads();
    const int rem = n - k - 1;
    for (int t = threadIdx.x; t < rem * rem; t += blockDim.x) {
      const int i = k + 1 + t % rem, j = k + 1 + t / rem;
      if (i >= j) A[(int64_t)j * ld + i] -= A[(int64_t)k * ld + i] * A[(int64_t)k * ld + j];
    }
    __syncthreads();
  }
  return 0;
}

// Column j of L^-1 (L lower, n x n, leading dimension ld) by forward substitution: out(i, j) for i >= j.
__device__ __forceinline__ void lower_inverse_column(const double* L, int n, int ld, int j, double* out, int ldo) {
  for (int i = 0; i < j; ++i) out[(int64_t)j * ldo + i] = 0.0;
  for (int i = j; i < n; ++i) {
    double s = i == j ? 1.0 : 0.0;
    for (int k = j; k < i; ++k) s -= L[(int64_t)k * ld + i] * out[(int64_t)j * ldo + k];
    out[(int64_t)j * ldo + i] = s / L[(int64_t)i * ld + i];
  }
}

// One pass of shifted CholeskyQR3 (Fukaya et al., SIAM J. Sci. Comput. 42, 2020) for both halves of every node of a
// level, from sym_tn_kernel's partial Gram matrices G = A_h^T A_h.  Pass 0 equilibrates the columns (d_q = |a_q|) and
// adds the shift 11 (m n + n (n + 1)) u |A D^-1|_2^2 (bounded by n); passes 1 and 2 are plain CholeskyQR.  G = L L^T,
// and the pass's R = L^T:
//   R^-1 slot <- (R D)^-1 (pass 0) or R^-1, the right factor sym_nn_kernel applies to A_h in place;
//   R slot    <- R D (pass 0) or R R_prev: the accumulated triangle with A_h(original) = Q_h R.
// status[node] = 1 (first failure kept) when a Gram matrix has no Cholesky factor: a zero, infinite or NaN column.
__global__ void __launch_bounds__(SY_THREADS) sym_qr_pass_kernel(const SymNode* __restrict__ nodes,
                                                                 const double* __restrict__ part, int nchunks,
                                                                 double* __restrict__ QR, int pass,
                                                                 int* __restrict__ status, int node_base) {
  extern __shared__ double sd[];  // the pass-0 column scales, r doubles
  const SymNode nd = nodes[blockIdx.x];
  const int n = nd.rank, r = nd.r;
  if (n == 0) return;
  for (int h = 0; h < 2; ++h) {
    const int nh = h ? nd.size - nd.half : nd.half;
    double* R = QR + nd.q_off + (int64_t)h * r * r;
    double* Ri = QR + nd.q_off + (int64_t)(2 + h) * r * r;
    double* G = QR + nd.q_off + (int64_t)(4 + h) * r * r;
    for (int t = threadIdx.x; t < n * n; t += SY_THREADS) {
      const int q = t % n, p = t / n;
      G[(int64_t)p * r + q] = sym_chunk_sum(part, blockIdx.x, h, nchunks, nh, r, r, q, p);
    }
    __syncthreads();
    if (pass == 0) {
      for (int q = threadIdx.x; q < n; q += SY_THREADS) sd[q] = sqrt(G[(int64_t)q * r + q]);
      __syncthreads();
      const double shift = 11.0 * ((double)nh * n + (double)n * (n + 1)) * 1.1102230246251565e-16 * n;
      for (int t = threadIdx.x; t < n * n; t += SY_THREADS) {
        const int q = t % n, p = t / n;
        G[(int64_t)p * r + q] = G[(int64_t)p * r + q] / (sd[q] * sd[p]) + (q == p ? shift : 0.0);
      }
      __syncthreads();
    }
    if (cta_cholesky(G, n, r) != 0) {
      if (threadIdx.x == 0 && status[node_base + blockIdx.x] == 0) status[node_base + blockIdx.x] = 1;
      return;
    }
    // R^-1 = L^-T: column j of L^-1 is row j of R^-1
    for (int j = threadIdx.x; j < n; j += SY_THREADS) {
      for (int i = 0; i < j; ++i) Ri[(int64_t)i * r + j] = 0.0;
      for (int i = j; i < n; ++i) {
        double s = i == j ? 1.0 : 0.0;
        for (int k = j; k < i; ++k) s -= G[(int64_t)k * r + i] * Ri[(int64_t)k * r + j];
        Ri[(int64_t)i * r + j] = s / G[(int64_t)i * r + i];
      }
      if (pass == 0)
        for (int i = j; i < n; ++i) Ri[(int64_t)i * r + j] /= sd[j];
    }
    // R accumulation, a thread per column c: new(q, c) = sum_{p = q..c} L(p, q) old(p, c), ascending q in place
    for (int c = threadIdx.x; c < n; c += SY_THREADS) {
      if (pass == 0) {
        for (int q = 0; q < n; ++q) R[(int64_t)c * r + q] = q <= c ? G[(int64_t)q * r + c] * sd[c] : 0.0;
      } else {
        for (int q = 0; q <= c; ++q) {
          double s = 0.0;
          for (int p = q; p <= c; ++p) s += G[(int64_t)q * r + p] * R[(int64_t)c * r + p];
          R[(int64_t)c * r + q] = s;
        }
      }
    }
    __syncthreads();
  }
}

// O[:, ocol0 + c] (+)= Q_h T_h[:, c] on both halves of every node of a level, c < ncols.  Q_h = the node's own columns
// of P, T_h(q, c) = T[b * tstride + h * thalf + q + c * ldt].  The CTA stages its rows of Q_h before it writes, and
// covers all columns of those rows, so O may be Q itself (accumulate = 0: Q_h <- A_h R^-1 in place).  Each entry is one
// sum over q in ascending order, whatever `rows` is.
// grid = (row chunk of `rows`, (node - b0) * 2 + h); rows a power of two <= SY_NN_ROWS; dynamic shared memory
// rows * (r + 1) doubles.
__global__ void __launch_bounds__(SY_THREADS) sym_nn_kernel(const SymNode* __restrict__ nodes, const double* P,
                                                            int64_t ldp, const double* __restrict__ T, int64_t tstride,
                                                            int64_t thalf, int ldt, double* O, int64_t ldo, int ocol0,
                                                            int ncols, int accumulate, int rows, int b0) {
  extern __shared__ double sa[];  // (row, q) at row * (rank + 1) + q
  const int b = b0 + (blockIdx.y >> 1);
  const SymNode nd = nodes[b];
  const int h = blockIdx.y & 1;
  const int rs = nd.start + (h ? nd.half : 0), nh = h ? nd.size - nd.half : nd.half;
  const int i0 = blockIdx.x * rows;
  const int n = nd.rank;
  if (i0 >= nh || n == 0) return;
  const int ni = min(rows, nh - i0);
  for (int t = threadIdx.x; t < rows * n; t += SY_THREADS) {
    const int i = t % rows, q = t / rows;
    sa[i * (n + 1) + q] = i < ni ? P[(int64_t)(nd.ucol + q) * ldp + rs + i0 + i] : 0.0;
  }
  __syncthreads();
  const double* Th = T + (int64_t)b * tstride + h * thalf;
  const int i = threadIdx.x % rows;
  if (i >= ni) return;
  const int nco = accumulate ? ncols : min(ncols, n);  // in place: the padding columns stay zero
  for (int c = threadIdx.x / rows; c < nco; c += SY_THREADS / rows) {
    const double* tc = Th + (int64_t)c * ldt;
    double acc = 0.0;
    for (int q = 0; q < n; ++q) acc += sa[i * (n + 1) + q] * tc[q];
    double* o = O + (int64_t)(ocol0 + c) * ldo + rs + i0 + i;
    *o = accumulate ? *o + acc : acc;
  }
}

// The node's 2r x 2r step once both halves are orthonormal (A_h = Q_h R_h):
//   I + M = I + [[0, R_0 R_1^T], [R_1 R_0^T, 0]] = L L^T   (padding: identity rows and columns, log 1 = 0),
//   X = L - I,  Y = L^-1 - I,  node_logdet = sum log L_kk.
// status[node] = 2 when I + M has no Cholesky factor: K~ is not positive definite.
__global__ void __launch_bounds__(SY_THREADS) sym_node_kernel(const SymNode* __restrict__ nodes,
                                                              const double* __restrict__ QR, double* __restrict__ XY,
                                                              double* __restrict__ node_logdet,
                                                              int* __restrict__ status, int node_base) {
  __shared__ double red[32];
  const SymNode nd = nodes[blockIdx.x];
  const int r = nd.r, n2 = 2 * r, n = nd.rank;
  double* X = XY + nd.x_off;
  double* Y = X + (int64_t)n2 * n2;
  if (n == 0 || status[node_base + blockIdx.x] != 0) {
    for (int t = threadIdx.x; t < 2 * n2 * n2; t += SY_THREADS) X[t] = 0.0;
    if (threadIdx.x == 0) node_logdet[node_base + blockIdx.x] = 0.0;
    return;
  }
  const double* R0 = QR + nd.q_off;
  const double* R1 = R0 + (int64_t)r * r;
  // lower triangle of I + M: entry (i, j), i >= r > j, is (R_1 R_0^T)(i - r, j) = sum_{p >= max(i - r, j)} R_1 R_0
  for (int t = threadIdx.x; t < n2 * n2; t += SY_THREADS) {
    const int i = t % n2, j = t / n2;
    double v = i == j ? 1.0 : 0.0;
    if (i >= r && j < r && i - r < n && j < n) {
      double s = 0.0;
      for (int p = max(i - r, j); p < n; ++p) s += R1[(int64_t)p * r + (i - r)] * R0[(int64_t)p * r + j];
      v = s;
    }
    X[t] = v;
  }
  __syncthreads();
  if (cta_cholesky(X, n2, n2) != 0) {
    if (threadIdx.x == 0) status[node_base + blockIdx.x] = 2;
    return;
  }
  double s = 0.0;
  for (int k = threadIdx.x; k < n2; k += SY_THREADS) s += log(X[(int64_t)k * n2 + k]);
  s = block_sum(s, red);
  if (threadIdx.x == 0) node_logdet[node_base + blockIdx.x] = s;
  for (int j = threadIdx.x; j < n2; j += SY_THREADS) lower_inverse_column(X, n2, n2, j, Y, n2);
  __syncthreads();
  for (int t = threadIdx.x; t < n2 * n2; t += SY_THREADS) {
    const int i = t % n2, j = t / n2;
    const double e = i == j ? 1.0 : 0.0;
    X[t] = i >= j ? X[t] - e : 0.0;
    Y[t] -= e;
  }
}

// T = S_op t for every node of a level, t = [Q_0^T B_0; Q_1^T B_1] (2r x ncols) summed from sym_tn_kernel's partials:
// S_op = X (op 0), X^T (op 1) or Y (op 2), all lower triangular before the transpose.  t goes to tbuf and T to ubuf,
// (2r x ncols) per node, leading dimension 2r.  One CTA per node.
__global__ void __launch_bounds__(SY_THREADS) sym_mid_kernel(const SymNode* __restrict__ nodes,
                                                             const double* __restrict__ part, int nchunks, int ncols,
                                                             const double* __restrict__ XY, int op,
                                                             double* __restrict__ tbuf, double* __restrict__ ubuf) {
  const SymNode nd = nodes[blockIdx.x];
  const int r = nd.r, n2 = 2 * r;
  if (nd.rank == 0) return;
  double* t = tbuf + (int64_t)blockIdx.x * n2 * ncols;
  double* u = ubuf + (int64_t)blockIdx.x * n2 * ncols;
  for (int e = threadIdx.x; e < n2 * ncols; e += SY_THREADS) {
    const int i = e % n2, c = e / n2, h = i >= r, q = i - h * r;
    const int nh = h ? nd.size - nd.half : nd.half;
    t[e] = q < nd.rank ? sym_chunk_sum(part, blockIdx.x, h, nchunks, nh, r, ncols, q, c) : 0.0;
  }
  __syncthreads();
  const double* S = XY + nd.x_off + (op == 2 ? (int64_t)n2 * n2 : 0);
  for (int e = threadIdx.x; e < n2 * ncols; e += SY_THREADS) {
    const int i = e % n2, c = e / n2;
    const double* tc = t + (int64_t)c * n2;
    double s = 0.0;
    if (op == 1) {
      for (int j = i; j < n2; ++j) s += S[(int64_t)i * n2 + j] * tc[j];
    } else {
      for (int j = 0; j <= i; ++j) s += S[(int64_t)j * n2 + i] * tc[j];
    }
    u[e] = s;
  }
}

// max |Q_h^T Q_h - I| over both halves of each node, from sym_tn_kernel's partial Gram matrices (a NaN counts as
// infinite).  out (may be null) receives it per node; with `status`, a node still marked 0 whose value is above `bar`
// is marked 3: its columns are too dependent for CholeskyQR, and sym_householder_kernel takes it over.
__global__ void __launch_bounds__(SY_THREADS) sym_orth_kernel(const SymNode* __restrict__ nodes,
                                                              const double* __restrict__ part, int nchunks,
                                                              double* __restrict__ out, int* __restrict__ status,
                                                              double bar, int node_base) {
  __shared__ double red[32];
  const SymNode nd = nodes[blockIdx.x];
  const int n = nd.rank;
  double m = 0.0;
  for (int h = 0; h < 2; ++h) {
    const int nh = h ? nd.size - nd.half : nd.half;
    for (int t = threadIdx.x; t < n * n; t += SY_THREADS) {
      const int q = t % n, p = t / n;
      const double e = fabs(sym_chunk_sum(part, blockIdx.x, h, nchunks, nh, nd.r, nd.r, q, p) - (q == p ? 1.0 : 0.0));
      m = (e <= m) ? m : (e == e ? e : __longlong_as_double(0x7ff0000000000000ll));
    }
  }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  m = warp_max(m);
  if (lane == 0) red[w] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    double v = 0.0;
    for (int k = 0; k < SY_THREADS / 32; ++k) v = fmax(v, red[k]);
    if (out) out[node_base + blockIdx.x] = v;
    if (status && n > 0 && status[node_base + blockIdx.x] == 0 && !(v <= bar)) status[node_base + blockIdx.x] = 3;
  }
}

// Householder QR of both halves of the nodes CholeskyQR could not orthonormalise (status 1: a Gram matrix without a
// Cholesky factor, 3: bases not orthonormal), one CTA per node, from the copy `A` of the level's columns taken before
// the CholeskyQR passes (column q at A + q * lda, global rows).  Rank-robust: Q = H_0 ... H_{n-1} [I; 0] is orthonormal
// to rounding whatever the conditioning, and A = Q R holds to rounding.  The reflectors overwrite A below the diagonal
// (LAPACK's dgeqr2 / dorg2r conventions), Q goes to the node's own columns of P and R to the node's R slot.  Each dot
// product is a warp's lanes added with a fixed butterfly, so the result is reproducible.  status <- 0, or 1 when a
// column is not finite; redone[node] <- 1 when the node's bases came from here.  Dynamic shared memory: r doubles.
__global__ void __launch_bounds__(SY_THREADS) sym_householder_kernel(const SymNode* __restrict__ nodes,
                                                                     double* __restrict__ A, int64_t lda,
                                                                     double* __restrict__ P, int64_t ldp,
                                                                     double* __restrict__ QR, int* __restrict__ status,
                                                                     int* __restrict__ redone, int node_base) {
  extern __shared__ double stau[];
  __shared__ double red[32];
  const SymNode nd = nodes[blockIdx.x];
  const int n = nd.rank, r = nd.r;
  const int st = status[node_base + blockIdx.x];
  if (n == 0 || (st != 1 && st != 3)) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = SY_THREADS / 32;
  bool finite = true;
  for (int h = 0; h < 2 && finite; ++h) {
    const int rs = nd.start + (h ? nd.half : 0), nh = h ? nd.size - nd.half : nd.half;
    double* a = A + (int64_t)nd.ucol * lda + rs;  // a(i, q) = a[q * lda + i]
    for (int k = 0; k < n; ++k) {
      double* ak = a + (int64_t)k * lda;
      double sg = 0.0;
      for (int i = k + 1 + threadIdx.x; i < nh; i += SY_THREADS) sg += ak[i] * ak[i];
      sg = block_sum(sg, red);
      const double alpha = ak[k];
      if (!isfinite(sg) || !isfinite(alpha)) { finite = false; break; }
      double tau = 0.0, beta = alpha, scal = 0.0;
      if (sg > 0.0) {
        const double norm = sqrt(alpha * alpha + sg);
        beta = alpha >= 0.0 ? -norm : norm;
        tau = (beta - alpha) / beta;
        scal = 1.0 / (alpha - beta);
      }
      __syncthreads();  // every thread has read alpha
      if (tau != 0.0)
        for (int i = k + 1 + threadIdx.x; i < nh; i += SY_THREADS) ak[i] *= scal;
      if (threadIdx.x == 0) { ak[k] = beta; stau[k] = tau; }
      __syncthreads();
      if (tau != 0.0) {
        for (int j = k + 1 + warp; j < n; j += nw) {  // A(k:, j) -= tau v (v^T A(k:, j)), v = [1; ak(k+1:)]
          double* aj = a + (int64_t)j * lda;
          double w = lane == 0 ? aj[k] : 0.0;
          for (int i = k + 1 + lane; i < nh; i += 32) w += ak[i] * aj[i];
          w = tau * warp_sum(w);
          if (lane == 0) aj[k] -= w;
          for (int i = k + 1 + lane; i < nh; i += 32) aj[i] -= w * ak[i];
        }
      }
      __syncthreads();
    }
    if (!finite) break;
    double* R = QR + nd.q_off + (int64_t)h * r * r;
    for (int t = threadIdx.x; t < n * n; t += SY_THREADS) {
      const int q = t % n, c = t / n;
      R[(int64_t)c * r + q] = q <= c ? a[(int64_t)c * lda + q] : 0.0;
    }
    double* Q = P + (int64_t)nd.ucol * ldp + rs;  // Q(i, j) = Q[j * ldp + i]
    for (int j = warp; j < n; j += nw)
      for (int i = lane; i < nh; i += 32) Q[(int64_t)j * ldp + i] = i == j ? 1.0 : 0.0;
    __syncthreads();
    for (int k = n - 1; k >= 0; --k) {
      const double tau = stau[k];
      const double* ak = a + (int64_t)k * lda;
      if (tau != 0.0) {
        for (int j = k + warp; j < n; j += nw) {  // columns < k are still e_j there
          double* qj = Q + (int64_t)j * ldp;
          double w = lane == 0 ? qj[k] : 0.0;
          for (int i = k + 1 + lane; i < nh; i += 32) w += ak[i] * qj[i];
          w = tau * warp_sum(w);
          if (lane == 0) qj[k] -= w;
          for (int i = k + 1 + lane; i < nh; i += 32) qj[i] -= w * ak[i];
        }
      }
      __syncthreads();
    }
  }
  if (threadIdx.x == 0) {
    status[node_base + blockIdx.x] = finite ? 0 : 1;
    redone[node_base + blockIdx.x] = 1;
  }
}

}  // namespace bgp
