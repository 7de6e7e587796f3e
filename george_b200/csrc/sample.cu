// sample.cu — draws from N(mean, C) on the device (GP.sample_conditional / GP.sample with a caller's generator):
// out = mean + z L^T, with z the caller's standard normals and L the lower Cholesky factor of sym(C) + jitter * I.
//
// The reference draws with numpy's multivariate_normal, an SVD of C on the host (src/george/utils.py:19-33).  Here the
// covariance stays on the device: it is symmetrised in place, factorised by the dense solver's Cholesky
// (dense_potrf_members) and multiplied by z either row by row (few draws: the product is a read of L per draw) or as
// a triangular GEMM on the DMMA pipe (many draws).  Every reduction adds in a fixed order: identical inputs give
// identical bits.
#include <algorithm>
#include <cmath>
#include <vector>

#include "linalg.cuh"

namespace bgp {

constexpr int SP_T = 32;  // tile of the symmetrisation

// A = sym(C) + jitter * I, exactly symmetric: CTA (bi, bj), bj <= bi, copies the tile of C's lower triangle
// (rows bi, columns bj; C[i*n + j], i >= j) onto the mirrored positions C[j*n + i] through shared memory, so both the
// read and the write are coalesced.  The positions written (i > j) are never read and the diagonal is read and written
// by the same thread, so the CTAs need no ordering.  A is its own transpose: column-major, as the Cholesky reads it.
// Member blockIdx.z works on C + blockIdx.z * cstride.
__global__ void __launch_bounds__(256) sample_sym_kernel(double* __restrict__ C, int64_t n, double jitter,
                                                         int64_t cstride) {
  const int64_t bi = blockIdx.y, bj = blockIdx.x;
  if (bj > bi) return;
  C += blockIdx.z * cstride;
  __shared__ double t[SP_T][SP_T + 1];
  const int tx = threadIdx.x & (SP_T - 1), ty = threadIdx.x / SP_T;
  for (int r = ty; r < SP_T; r += 256 / SP_T) {
    const int64_t i = bi * SP_T + r, j = bj * SP_T + tx;
    if (i < n && j <= i) t[r][tx] = C[i * n + j];
  }
  __syncthreads();
  for (int r = ty; r < SP_T; r += 256 / SP_T) {
    const int64_t j = bj * SP_T + r, i = bi * SP_T + tx;  // write row j, column i: C's element (i, j)
    if (i >= n || j > i) continue;
    C[j * n + i] = (i == j) ? t[tx][r] + jitter : t[tx][r];
  }
}

// zero the strict upper triangle of the column-major factor (entries (i, j), i < j, at L[j*n + i]), which the
// factorisation leaves holding A, so that the product may read whole tiles of L; member blockIdx.z at L + z * lstride
__global__ void sample_zero_upper_kernel(double* __restrict__ L, int64_t n, int64_t lstride) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  L += blockIdx.z * lstride;
  for (int64_t j = blockIdx.y; j < n; j += gridDim.y)
    if (i < j) L[j * n + i] = 0.0;
}

// few draws: out[a][j] = mean[j] + sum_{i<=j} z[a][i] L[j][i], the arithmetic of apply_sqrt_kernel (dense.cu) plus the
// mean; one thread per output entry, the row of L it needs read coalesced across the CTA.  Member blockIdx.z reads
// L + z * lstride, mean + z * mstride and z, out + z * zstride.
__global__ void sample_rows_kernel(const double* __restrict__ L, int64_t n, const double* __restrict__ z,
                                   const double* __restrict__ mean, double* __restrict__ out, int64_t lstride,
                                   int64_t mstride, int64_t zstride) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t a = blockIdx.y, m = blockIdx.z;
  if (j >= n) return;
  L += m * lstride; mean += m * mstride; z += m * zstride; out += m * zstride;
  double s = 0.0;
  for (int64_t i = 0; i <= j; ++i) s += z[a * n + i] * L[i * n + j];  // L[j][i] column-major = L[i*n + j]
  out[a * n + j] = mean[j] + s;
}

// many draws, the operands of gemm_dmma's C -= A'B': out starts as the mean in every row and z is negated (exactly);
// member blockIdx.z on z, out + z * total (its size x n draws) and mean + z * mstride
__global__ void sample_dmma_operands_kernel(double* __restrict__ z, const double* __restrict__ mean,
                                            double* __restrict__ out, int64_t n, int64_t total, int64_t mstride) {
  z += blockIdx.z * total; out += blockIdx.z * total; mean += blockIdx.z * mstride;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (int64_t)gridDim.x * blockDim.x) {
    z[p] = -z[p];
    out[p] = mean[p % n];
  }
}

// device-event timing of the last successful draw on this thread (bgp_sample_last_timing): events 0..3 mark the start
// of the covariance, of the factorisation (symmetrisation included), of the product and its end
namespace {
struct SampleTiming {
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  double ms[3] = {0, 0, 0};
};
thread_local SampleTiming g_sample_timing;
}  // namespace

int sample_mark(int i, cudaStream_t s) {
  cudaEvent_t& e = g_sample_timing.ev[i];
  if (!e) BGP_CUDA(cudaEventCreate(&e));
  BGP_CUDA(cudaEventRecord(e, s));
  return BGP_OK;
}

int mvn_sample_check(int64_t ns, int64_t size, double jitter) {
  if (ns < 0) { set_error("negative number of test points"); return BGP_ERR_INVALID; }
  if (size < 0) { set_error("negative number of draws"); return BGP_ERR_INVALID; }
  if (!(jitter >= 0.0) || !std::isfinite(jitter)) { set_error("jitter must be finite and >= 0"); return BGP_ERR_INVALID; }
  return BGP_OK;
}

int mvn_factor_members(double* C, int64_t ns, double jitter, int members, int* info, const int* gemm_info,
                       DevBuf<GemmDesc>& gdesc, cudaStream_t s) {
  const unsigned T = (unsigned)((ns + SP_T - 1) / SP_T);
  sample_sym_kernel<<<dim3(T, T, (unsigned)members), 256, 0, s>>>(C, ns, jitter, ns * ns);
  BGP_LAUNCH_CHECK();
  BGP_CUDA(cudaMemsetAsync(info, 0, sizeof(int) * members, s));
  return dense_potrf_members(C, ns, ns * ns, members, info, gemm_info, gdesc, s);
}

int64_t mvn_product_descs(int64_t ns, int64_t size) {
  if (size < BGP_SAMPLE_DMMA_ROWS) return 0;
  const int64_t slab = std::min<int64_t>(size, (int64_t)65535 * GD_BN);
  return (size + slab - 1) / slab * ((ns + GD_BM - 1) / GD_BM);
}

int mvn_product_members(double* C, int64_t ns, const double* mean, int64_t mstride, double* z, int64_t size,
                        double* out, int members, DevBuf<GemmDesc>& gdesc, cudaStream_t s) {
  const unsigned mb = (unsigned)members;
  const int64_t total = size * ns;  // a member's draws
  sample_zero_upper_kernel<<<dim3((unsigned)((ns + 255) / 256), (unsigned)std::min<int64_t>(ns, 65535), mb), 256, 0,
                             s>>>(C, ns, ns * ns);
  BGP_LAUNCH_CHECK();
  if (size < BGP_SAMPLE_DMMA_ROWS) {
    sample_rows_kernel<<<dim3((unsigned)((ns + 127) / 128), (unsigned)size, mb), 128, 0, s>>>(C, ns, z, mean, out,
                                                                                              ns * ns, mstride, total);
    BGP_LAUNCH_CHECK();
    return BGP_OK;
  }
  sample_dmma_operands_kernel<<<dim3((unsigned)std::min<int64_t>((total + 255) / 256, 4096), 1, mb), 256, 0, s>>>(
      z, mean, out, ns, total, mstride);
  BGP_LAUNCH_CHECK();
  // column-major view: out^T (ns x size, ld ns) -= L (-z)^T.  One descriptor per member, per 128 rows of out^T (= 128
  // columns of out) and per slab of at most 65535 * 128 draws (the grid's y limit); the tile of rows j0.. stops K at
  // its last row, so the blocks of L above the diagonal are neither read nor multiplied.  Every member's descriptors
  // have the geometry of a single draw's, so its bits do not depend on the number of members.
  const int64_t slab = std::min<int64_t>(size, (int64_t)65535 * GD_BN);
  std::vector<GemmDesc> descs;
  for (int m = 0; m < members; ++m) {
    const double* Lm = C + m * ns * ns;
    double* zm = z + m * total;
    double* om = out + m * total;
    for (int64_t a0 = 0; a0 < size; a0 += slab)
      for (int64_t j0 = 0; j0 < ns; j0 += GD_BM) {
        GemmDesc d;
        d.A = Lm + j0; d.lda = ns;                // A'(m, k) = L[j0 + m][k] = C[k*ns + j0 + m]
        d.B = zm + a0 * ns; d.ldb = ns;           // B'(k, a) = -z[a0 + a][k]
        d.C = om + a0 * ns + j0; d.ldc = ns;      // C(m, a) = out[a0 + a][j0 + m]
        d.M = (int)std::min<int64_t>(GD_BM, ns - j0);
        d.N = (int)std::min(slab, size - a0);
        d.K = (int)std::min<int64_t>(j0 + GD_BM, ns);
        d.mode = GD_SUB;
        descs.push_back(d);
      }
  }
  BGP_TRY(gdesc.reserve(descs.size(), s));
  BGP_CUDA(cudaMemcpyAsync(gdesc.p, descs.data(), sizeof(GemmDesc) * descs.size(), cudaMemcpyHostToDevice, s));
  // descs is pageable host memory: the copy above has been staged before cudaMemcpyAsync returned
  return gemm_dmma_launch<false, true>(gdesc.p, (int)descs.size(), GD_BM, (int)slab, nullptr, s);
}

int mvn_draw_dev(double* C, int64_t ns, const double* mean, double* z, int64_t size, double jitter, double* out,
                 DevBuf<int>& info, DevBuf<GemmDesc>& gdesc, cudaStream_t s) {
  if (ns == 0 || size == 0) return BGP_OK;
  BGP_TRY(sample_mark(1, s));
  BGP_TRY(info.reserve(1, s));
  BGP_TRY(mvn_factor_members(C, ns, jitter, 1, info.p, info.p, gdesc, s));
  BGP_TRY(sample_mark(2, s));
  int h_info = 0;
  BGP_CUDA(cudaMemcpyAsync(&h_info, info.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  if (h_info != 0) {
    set_error("%d-th leading minor of the array is not positive definite (a larger jitter adds more to the diagonal)",
              h_info);
    return BGP_ERR_LINALG;
  }
  BGP_TRY(mvn_product_members(C, ns, mean, 0, z, size, out, 1, gdesc, s));
  return sample_mark(3, s);
}

// mvn_draw_dev with mean and z from the host and the draws copied back: the common tail of bgp_mvn_sample,
// bgp_dense_sample and bgp_hodlr_sample.  C (ns x ns) is on the device already.  Workspace: (2 size + 1) ns doubles.
int mvn_draw_host_io(double* C, int64_t ns, const double* mean, const double* z, int64_t size, double jitter,
                     double* out, cudaStream_t s) {
  if (ns == 0 || size == 0) return BGP_OK;
  DevBuf<double> dm, dz, dout;
  DevBuf<int> info;
  DevBuf<GemmDesc> gdesc;
  BGP_TRY(dm.alloc((size_t)ns, s));
  BGP_TRY(dz.alloc((size_t)size * ns, s));
  BGP_TRY(dout.alloc((size_t)size * ns, s));
  BGP_CUDA(cudaMemcpyAsync(dm.p, mean, sizeof(double) * ns, cudaMemcpyHostToDevice, s));
  BGP_CUDA(cudaMemcpyAsync(dz.p, z, sizeof(double) * size * ns, cudaMemcpyHostToDevice, s));
  BGP_TRY(mvn_draw_dev(C, ns, dm.p, dz.p, size, jitter, dout.p, info, gdesc, s));
  BGP_CUDA(cudaMemcpyAsync(out, dout.p, sizeof(double) * size * ns, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  for (int i = 0; i < 3; ++i) {
    float ms = 0;
    cudaEventElapsedTime(&ms, g_sample_timing.ev[i], g_sample_timing.ev[i + 1]);
    g_sample_timing.ms[i] = ms;
  }
  return BGP_OK;
}

}  // namespace bgp

using namespace bgp;

extern "C" {

int bgp_mvn_sample(const double* cov, int64_t ns, const double* mean, const double* z, int64_t size, double jitter,
                   double* out) {
  BGP_TRY(mvn_sample_check(ns, size, jitter));
  if (ns == 0 || size == 0) return BGP_OK;
  BGP_TRY(require_device());
  cudaStream_t s = 0;
  DevBuf<double> dC;
  BGP_TRY(dC.alloc((size_t)ns * ns, s));
  BGP_TRY(sample_mark(0, s));
  BGP_CUDA(cudaMemcpyAsync(dC.p, cov, sizeof(double) * ns * ns, cudaMemcpyHostToDevice, s));
  return mvn_draw_host_io(dC.p, ns, mean, z, size, jitter, out, s);
}

int bgp_sample_last_timing(double* ms3) {
  for (int i = 0; i < 3; ++i) ms3[i] = g_sample_timing.ms[i];
  return BGP_OK;
}

}  // extern "C"
