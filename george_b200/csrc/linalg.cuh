// linalg.cuh — dense linear-algebra routines shared between translation units (dense.cu, sample.cu, hodlr.cu).
#pragma once

#include "common.cuh"
#include "gemm_dmma.cuh"

namespace bgp {

// Blocked right-looking Cholesky of `members` column-major n x n matrices (member m at A + m * mstride), lower factor
// in place; info[m] = k+1 for the first pivot that is not positive (NaN included), as LAPACK's dpotrf.  gemm_info: the
// word the trailing updates test before running (a single factorisation passes its info word).  dense.cu.
int dense_potrf_members(double* A, int64_t n, int64_t mstride, int members, int* info, const int* gemm_info,
                        DevBuf<GemmDesc>& gdesc, cudaStream_t s);

// out = mean + z L^T with L the lower Cholesky factor of A = sym(C) + jitter * I, all on the device (sample.cu).
//   C     ns x ns row-major; its lower triangle C[i*ns + j], i >= j, defines sym(C).  Overwritten by L.
//   mean  ns;  z  size x ns row-major (overwritten: negated on the many-row path);  out  size x ns row-major.
// BGP_ERR_LINALG ("%d-th leading minor ...") when A is not positive definite; nothing is written to out then.
int mvn_draw_dev(double* C, int64_t ns, const double* mean, double* z, int64_t size, double jitter, double* out,
                 DevBuf<int>& info, DevBuf<GemmDesc>& gdesc, cudaStream_t s);
// The two halves of mvn_draw_dev for `members` draws at once, one launch per step for all of them (member m: C + m ns^2,
// mean + m * mstride, z and out + m * size * ns); mvn_draw_dev runs them with one member and checks info in between.
//   mvn_factor_members: A_m = sym(C_m) + jitter * I factorised in place, info[m] its dpotrf index (gemm_info as in
//     dense_potrf_members: a batch passes nullptr, so a failed member's steps run on its own slab only).
//   mvn_product_members: zero the upper triangles, then out = mean + z L^T (rows below BGP_SAMPLE_DMMA_ROWS draws, the
//     DMMA GEMM from it with mvn_product_descs(ns, size) descriptors per member, uploaded to gdesc).
int mvn_factor_members(double* C, int64_t ns, double jitter, int members, int* info, const int* gemm_info,
                       DevBuf<GemmDesc>& gdesc, cudaStream_t s);
int mvn_product_members(double* C, int64_t ns, const double* mean, int64_t mstride, double* z, int64_t size,
                        double* out, int members, DevBuf<GemmDesc>& gdesc, cudaStream_t s);
int64_t mvn_product_descs(int64_t ns, int64_t size);
// mvn_draw_dev with mean, z and out on the host (synchronises s)
int mvn_draw_host_io(double* C, int64_t ns, const double* mean, const double* z, int64_t size, double jitter,
                     double* out, cudaStream_t s);
// records timing event i (0: covariance start, 1: factorisation start, 2: product start, 3: end) on s for
// bgp_sample_last_timing
int sample_mark(int i, cudaStream_t s);
// the argument checks of the sampling entries: BGP_ERR_INVALID for ns < 0, size < 0, a negative or non-finite jitter
int mvn_sample_check(int64_t ns, int64_t size, double jitter);

}  // namespace bgp
