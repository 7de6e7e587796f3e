// hodlr_sym.cu — the symmetric factor K~ = W W^T of a computed HODLR factorisation (kernels: hodlr_sym.cuh).
//
// Build (sym_build), from what compute() left on the device: the leaves' L D L^T and the raw ACA factors of every node
// (the V panel, which the up-sweep never modifies):
//   1. copy each level's used V columns into the packed panel P (the U panel's column layout, zero padding);
//   2. P <- D^-1/2 L^-1 P on the leaf rows (each leaf over its ancestors' columns);
//   3. per level, deepest first: orthonormalise the node's own columns on both halves (equilibrated, shifted
//      CholeskyQR3: three passes of Gram -> Cholesky -> triangular product, rows-parallel; a node whose bases then
//      miss SY_ORTH_BAR, or whose Gram matrix had no Cholesky factor, is redone by Householder QR from a copy of its
//      columns taken before the passes: ACA columns can be numerically dependent, e.g. a block the ACA returned
//      dense, which no Gram-based method resolves), factor
//      I + M = L L^T (2r x 2r), keep X = L - I and Y = L^-1 - I, and apply W_v^-1 = I + Q Y Q^T to the ancestor
//      columns on the node's rows.
// log|K~| = sum log D_ii + 2 sum_v sum log diag L_v.
// Apply (sym_apply), in groups of 64 columns: root to deepest Z += Q X Q^T Z, then Z <- L D^1/2 Z on the leaves; the
// transpose runs the reverse order with X^T and D^1/2 L^T.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "hodlr_sym.cuh"

namespace bgp {

struct SymLevelHost {
  int r = 0, ucol = 0, vcol = 0, node0 = 0, nn = 0, max_size = 0, max_half = 0;
  int64_t q_base = 0, x_base = 0;
};

struct SymFactor {
  int64_t n = 0;
  int rtot = 0, max_leaf = 0;
  std::vector<SymLevelHost> levels;
  std::vector<SymNode> nodes;   // level by level, deepest level last
  std::vector<int> node_id;     // pre-order id of each entry of `nodes`
  std::vector<SymLeaf> leaves;
  const double* dL = nullptr;   // the handle's leaf factors (valid while the factorisation is)
  double logdet = 0.0;
  DevBuf<SymNode> d_nodes;
  DevBuf<SymLeaf> d_leaves;
  DevBuf<double> P, XY, QR, part, tbuf, ubuf, z, leaf_logdet, node_logdet, orth, acopy;
  DevBuf<int> status, bad_row, redone;
  std::vector<int> householder_nodes;  // per level: nodes whose bases came from sym_householder_kernel
  cudaEvent_t ev[2] = {nullptr, nullptr};
  double build_ms = 0.0, apply_ms = 0.0;  // device time of the last build / of the last apply's products
  ~SymFactor() {
    for (cudaEvent_t e : ev)
      if (e) cudaEventDestroy(e);
  }
};

// |Q^T Q - I| above which CholeskyQR3's bases are redone by Householder QR (the factor identity's 1e-13 target)
constexpr double SY_ORTH_BAR = 1e-13;
// The largest level rank the build accepts.  Each node's 2r x 2r Cholesky of I + M, its triangular inverse and the
// Householder QR of its halves run in one CTA, in time that grows as r^3 (DESIGN.md: 1.9 s at r = 800, 3.9 s at 1024 on
// one H100); past this the build is rejected before it launches anything.
constexpr int SY_MAX_RANK = 2048;
// nodes per launch of the kernels that put the node on gridDim.y (at most 65535; sym_tn / sym_nn use node * 2 + half)
constexpr int SY_LEVEL_SLAB = 32767;

SymFactor* sym_create() { return new SymFactor(); }
void sym_destroy(SymFactor* f) { delete f; }

static const size_t SY_SMEM_MAX = 200 * 1024;

static void set_sym_func_attrs() {
  static std::atomic<uint64_t> done{0};
  int dev = 0;
  cudaGetDevice(&dev);
  const uint64_t bit = dev < 64 ? (1ull << dev) : 0;
  if (bit && (done.load(std::memory_order_relaxed) & bit)) return;
  cudaFuncSetAttribute(sym_leaf_forward_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SY_SMEM_MAX);
  cudaFuncSetAttribute(sym_leaf_forward_kernel<SY_LEAF_COLS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SY_SMEM_MAX);
  cudaFuncSetAttribute(sym_leaf_product_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SY_SMEM_MAX);
  cudaFuncSetAttribute(sym_leaf_product_kernel<SY_LEAF_COLS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                       (int)SY_SMEM_MAX);
  cudaFuncSetAttribute(sym_nn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SY_SMEM_MAX);
  done.fetch_or(bit, std::memory_order_relaxed);
}

// the leaf kernels stage (max_leaf x cols) doubles: 8 columns for leaves of up to 3200 rows, one column beyond
static int leaf_cols(int max_leaf) {
  return sizeof(double) * (size_t)max_leaf * SY_LEAF_COLS <= SY_SMEM_MAX ? SY_LEAF_COLS : 1;
}

static int launch_leaf_forward(SymFactor* f, cudaStream_t s) {
  int maxc = 0;
  for (const SymLeaf& lf : f->leaves) maxc = std::max(maxc, lf.ncols);
  if (maxc == 0 || f->leaves.empty()) return BGP_OK;
  const int cols = leaf_cols(f->max_leaf), ngroups = (maxc + cols - 1) / cols;
  const dim3 grid((unsigned)(f->leaves.size() * (size_t)ngroups));
  const size_t smem = sizeof(double) * (size_t)f->max_leaf * cols;
  if (cols == SY_LEAF_COLS)
    sym_leaf_forward_kernel<SY_LEAF_COLS><<<grid, SY_THREADS, smem, s>>>(f->d_leaves.p, f->dL, f->P.p, f->n,
                                                                          f->max_leaf, ngroups);
  else
    sym_leaf_forward_kernel<1><<<grid, SY_THREADS, smem, s>>>(f->d_leaves.p, f->dL, f->P.p, f->n, f->max_leaf, ngroups);
  BGP_LAUNCH_CHECK();
  return BGP_OK;
}

static int launch_leaf_product(SymFactor* f, double* Z, int nc, int transpose, cudaStream_t s) {
  const int cols = leaf_cols(f->max_leaf), ngroups = (nc + cols - 1) / cols;
  const dim3 grid((unsigned)(f->leaves.size() * (size_t)ngroups));
  const size_t smem = sizeof(double) * (size_t)f->max_leaf * cols;
  if (cols == SY_LEAF_COLS)
    sym_leaf_product_kernel<SY_LEAF_COLS><<<grid, SY_THREADS, smem, s>>>(f->d_leaves.p, f->dL, Z, f->n, nc,
                                                                          f->max_leaf, ngroups, transpose);
  else
    sym_leaf_product_kernel<1><<<grid, SY_THREADS, smem, s>>>(f->d_leaves.p, f->dL, Z, f->n, nc, f->max_leaf, ngroups,
                                                               transpose);
  BGP_LAUNCH_CHECK();
  return BGP_OK;
}

static int nchunks_of(const SymLevelHost& L) { return std::max(1, (L.max_half + 1 + SY_TN_CHUNK - 1) / SY_TN_CHUNK); }

// partial products Q_h^T B_h of every node of level L, for columns [bcol0, bcol0 + ncols) of B
static int launch_tn(SymFactor* f, const SymLevelHost& L, const double* B, int bcol0, int ncols, cudaStream_t s) {
  const int nch = nchunks_of(L);
  BGP_TRY(f->part.reserve((size_t)L.nn * 2 * nch * L.r * ncols, s));
  for (int b0 = 0; b0 < L.nn; b0 += SY_LEVEL_SLAB) {
    const int nb = std::min(SY_LEVEL_SLAB, L.nn - b0);
    const dim3 grid((unsigned)nch, (unsigned)(2 * nb), (unsigned)((ncols + SY_TN_TC - 1) / SY_TN_TC));
    sym_tn_kernel<<<grid, SY_THREADS, 0, s>>>(f->d_nodes.p + L.node0, f->P.p, f->n, B, f->n, bcol0, ncols, f->part.p, nch,
                                              b0);
    BGP_LAUNCH_CHECK();
  }
  return BGP_OK;
}

// sym_nn_kernel's rows per CTA: 32, halved until the staged rows x (r + 1) doubles fit (one row up to r = 25599)
static int nn_rows(int r) {
  int rows = SY_NN_ROWS;
  while (rows > 1 && sizeof(double) * (size_t)rows * (r + 1) > SY_SMEM_MAX) rows /= 2;
  return rows;
}

static int launch_nn(SymFactor* f, const SymLevelHost& L, const double* T, int64_t tstride, int64_t thalf, int ldt,
                     double* O, int ocol0, int ncols, int accumulate, cudaStream_t s) {
  const int rows = nn_rows(L.r);
  const size_t smem = sizeof(double) * rows * (size_t)(L.r + 1);
  for (int b0 = 0; b0 < L.nn; b0 += SY_LEVEL_SLAB) {
    const int nb = std::min(SY_LEVEL_SLAB, L.nn - b0);
    const dim3 grid((unsigned)((L.max_half + 1 + rows - 1) / rows), (unsigned)(2 * nb));
    sym_nn_kernel<<<grid, SY_THREADS, smem, s>>>(f->d_nodes.p + L.node0, f->P.p, f->n, T, tstride, thalf, ldt, O, f->n,
                                                 ocol0, ncols, accumulate, rows, b0);
    BGP_LAUNCH_CHECK();
  }
  return BGP_OK;
}

// Z[:, 0:ncols] += Q_v S_op Q_v^T Z on every node of level L (op: 0 = X, 1 = X^T, 2 = Y)
static int level_apply(SymFactor* f, const SymLevelHost& L, double* Z, int ncols, int op, cudaStream_t s) {
  if (L.r == 0 || ncols == 0) return BGP_OK;
  BGP_TRY(launch_tn(f, L, Z, 0, ncols, s));
  const size_t tsz = (size_t)L.nn * 2 * L.r * ncols;
  BGP_TRY(f->tbuf.reserve(tsz, s));
  BGP_TRY(f->ubuf.reserve(tsz, s));
  sym_mid_kernel<<<L.nn, SY_THREADS, 0, s>>>(f->d_nodes.p + L.node0, f->part.p, nchunks_of(L), ncols, f->XY.p, op,
                                             f->tbuf.p, f->ubuf.p);
  BGP_LAUNCH_CHECK();
  return launch_nn(f, L, f->ubuf.p, (int64_t)2 * L.r * ncols, L.r, 2 * L.r, Z, 0, ncols, 1, s);
}

int sym_build(SymFactor* f, int64_t n, int nlev, const int* lev, const int* nodes, int nleaf, const int64_t* leaves,
              int max_leaf, const double* dL, const double* V, int64_t ldv, cudaStream_t s, double* logdet_out) {
  set_sym_func_attrs();
  f->n = n; f->max_leaf = max_leaf; f->dL = dL;
  f->levels.assign(nlev, SymLevelHost());
  f->nodes.clear(); f->node_id.clear(); f->leaves.clear();
  // per level: r, ucol, vcol, node count; per node (level order): start, size, half, rank, pre-order id
  int64_t q_total = 0, x_total = 0;
  f->rtot = 0;
  for (int l = 0, k = 0; l < nlev; ++l) {
    SymLevelHost& L = f->levels[l];
    L.r = lev[4 * l]; L.ucol = lev[4 * l + 1]; L.vcol = lev[4 * l + 2]; L.nn = lev[4 * l + 3];
    L.node0 = (int)f->nodes.size();
    L.q_base = q_total; L.x_base = x_total;
    f->rtot = std::max(f->rtot, L.ucol + L.r);
    for (int b = 0; b < L.nn; ++b, ++k) {
      const int* e = nodes + 5 * k;
      SymNode d;
      d.start = e[0]; d.size = e[1]; d.half = e[2]; d.rank = e[3]; d.r = L.r; d.ucol = L.ucol;
      d.q_off = q_total; d.x_off = x_total;
      q_total += (int64_t)6 * L.r * L.r;
      x_total += (int64_t)2 * (2 * L.r) * (2 * L.r);
      L.max_size = std::max(L.max_size, d.size);
      L.max_half = std::max(L.max_half, d.size - d.half);
      f->nodes.push_back(d);
      f->node_id.push_back(e[4]);
    }
  }
  for (int i = 0; i < nleaf; ++i) {
    SymLeaf lf;
    lf.start = (int)leaves[4 * i]; lf.size = (int)leaves[4 * i + 1]; lf.ncols = (int)leaves[4 * i + 2]; lf._pad = 0;
    lf.off = leaves[4 * i + 3];
    f->leaves.push_back(lf);
  }
  const int nn = (int)f->nodes.size();
  for (int l = 0; l < nlev; ++l) {  // before anything is launched
    const SymLevelHost& L = f->levels[l];
    if (L.r <= SY_MAX_RANK) continue;
    int k = L.node0;
    while (k + 1 < L.node0 + L.nn && f->nodes[k].rank <= SY_MAX_RANK) ++k;
    const SymNode& d = f->nodes[k];
    set_error("HODLR node %d (rows [%d, %d), level %d) has rank %d, above the symmetric factor's limit of %d",
              f->node_id[k], d.start, d.start + d.size, l, d.rank, SY_MAX_RANK);
    return BGP_ERR_INVALID;
  }
  // BGP_SYM_QR=householder (diagnostic): every node through the Householder QR, none through CholeskyQR3
  const char* qr_env = getenv("BGP_SYM_QR");
  const bool all_householder = qr_env && !strcmp(qr_env, "householder");
  BGP_TRY(f->d_nodes.reserve(std::max(nn, 1), s));
  BGP_TRY(f->d_leaves.reserve(std::max(nleaf, 1), s));
  BGP_TRY(f->P.reserve((size_t)n * std::max(f->rtot, 1), s));
  BGP_TRY(f->QR.reserve((size_t)std::max<int64_t>(q_total, 1), s));
  BGP_TRY(f->XY.reserve((size_t)std::max<int64_t>(x_total, 1), s));
  BGP_TRY(f->leaf_logdet.reserve(std::max(nleaf, 1), s));
  BGP_TRY(f->node_logdet.reserve(std::max(nn, 1), s));
  BGP_TRY(f->status.reserve(std::max(nn, 1), s));
  BGP_TRY(f->redone.reserve(std::max(nn, 1), s));
  BGP_TRY(f->bad_row.reserve(1, s));
  if (nn) BGP_CUDA(cudaMemcpyAsync(f->d_nodes.p, f->nodes.data(), sizeof(SymNode) * nn, cudaMemcpyHostToDevice, s));
  BGP_CUDA(cudaMemcpyAsync(f->d_leaves.p, f->leaves.data(), sizeof(SymLeaf) * nleaf, cudaMemcpyHostToDevice, s));
  BGP_CUDA(cudaMemsetAsync(f->status.p, 0, sizeof(int) * std::max(nn, 1), s));
  BGP_CUDA(cudaMemsetAsync(f->redone.p, 0, sizeof(int) * std::max(nn, 1), s));
  BGP_CUDA(cudaMemsetAsync(f->node_logdet.p, 0, sizeof(double) * std::max(nn, 1), s));  // levels of rank 0 add nothing
  const int no_row = 0x7fffffff;
  BGP_CUDA(cudaMemcpyAsync(f->bad_row.p, &no_row, sizeof(int), cudaMemcpyHostToDevice, s));

  if (!f->ev[0]) {
    BGP_CUDA(cudaEventCreate(&f->ev[0]));
    BGP_CUDA(cudaEventCreate(&f->ev[1]));
  }
  int max_r = 1;
  for (const SymLevelHost& L : f->levels) max_r = std::max(max_r, L.r);
  BGP_TRY(f->acopy.reserve((size_t)n * max_r, s));
  BGP_CUDA(cudaEventRecord(f->ev[0], s));
  // 1. P <- the used V columns
  for (const SymLevelHost& L : f->levels) {
    if (L.r == 0) continue;
    for (int b0 = 0; b0 < L.nn; b0 += SY_LEVEL_SLAB) {
      const int nb = std::min(SY_LEVEL_SLAB, L.nn - b0);
      sym_copy_kernel<<<dim3((unsigned)((L.max_size + SY_THREADS - 1) / SY_THREADS), (unsigned)nb), SY_THREADS, 0, s>>>(
          f->d_nodes.p + L.node0 + b0, V, ldv, L.vcol, f->P.p, n);
      BGP_LAUNCH_CHECK();
    }
  }
  // 2. leaves: D > 0, log|D|, P <- D^-1/2 L^-1 P
  sym_leaf_check_kernel<<<nleaf, SY_THREADS, 0, s>>>(f->d_leaves.p, dL, f->leaf_logdet.p, f->bad_row.p);
  BGP_LAUNCH_CHECK();
  BGP_TRY(launch_leaf_forward(f, s));
  // 3. levels, deepest first
  for (int l = nlev - 1; l >= 0; --l) {
    const SymLevelHost& L = f->levels[l];
    if (L.r == 0) continue;
    BGP_CUDA(cudaMemcpyAsync(f->acopy.p, f->P.p + (int64_t)L.ucol * n, sizeof(double) * n * L.r,
                             cudaMemcpyDeviceToDevice, s));
    for (int pass = 0; pass < (all_householder ? 0 : 3); ++pass) {
      BGP_TRY(launch_tn(f, L, f->P.p, L.ucol, L.r, s));
      sym_qr_pass_kernel<<<L.nn, SY_THREADS, sizeof(double) * L.r, s>>>(f->d_nodes.p + L.node0, f->part.p,
                                                                        nchunks_of(L), f->QR.p, pass, f->status.p,
                                                                        L.node0);
      BGP_LAUNCH_CHECK();
      const int64_t rr = (int64_t)L.r * L.r;
      BGP_TRY(launch_nn(f, L, f->QR.p + L.q_base + 2 * rr, 6 * rr, rr, L.r, f->P.p, L.ucol, L.r, 0, s));
    }
    BGP_TRY(launch_tn(f, L, f->P.p, L.ucol, L.r, s));
    // (all_householder: a bar below every |Q^T Q - I| marks every node of nonzero rank)
    sym_orth_kernel<<<L.nn, SY_THREADS, 0, s>>>(f->d_nodes.p + L.node0, f->part.p, nchunks_of(L), nullptr, f->status.p,
                                                all_householder ? -1.0 : SY_ORTH_BAR, L.node0);
    BGP_LAUNCH_CHECK();
    // (the copy's column q sits at acopy + q n: shift the base so that the kernel's column ucol + q lands there)
    sym_householder_kernel<<<L.nn, SY_THREADS, sizeof(double) * L.r, s>>>(
        f->d_nodes.p + L.node0, f->acopy.p - (int64_t)L.ucol * n, n, f->P.p, n, f->QR.p, f->status.p, f->redone.p,
        L.node0);
    BGP_LAUNCH_CHECK();
    sym_node_kernel<<<L.nn, SY_THREADS, 0, s>>>(f->d_nodes.p + L.node0, f->QR.p, f->XY.p, f->node_logdet.p,
                                                f->status.p, L.node0);
    BGP_LAUNCH_CHECK();
    if (L.ucol > 0) {  // W_v^-1 on the ancestor columns
      BGP_TRY(launch_tn(f, L, f->P.p, 0, L.ucol, s));
      const size_t tsz = (size_t)L.nn * 2 * L.r * L.ucol;
      BGP_TRY(f->tbuf.reserve(tsz, s));
      BGP_TRY(f->ubuf.reserve(tsz, s));
      sym_mid_kernel<<<L.nn, SY_THREADS, 0, s>>>(f->d_nodes.p + L.node0, f->part.p, nchunks_of(L), L.ucol, f->XY.p, 2,
                                                 f->tbuf.p, f->ubuf.p);
      BGP_LAUNCH_CHECK();
      BGP_TRY(launch_nn(f, L, f->ubuf.p, (int64_t)2 * L.r * L.ucol, L.r, 2 * L.r, f->P.p, 0, L.ucol, 1, s));
    }
  }

  BGP_CUDA(cudaEventRecord(f->ev[1], s));
  // errors and the log-determinant
  int bad_row = no_row;
  std::vector<int> status(nn), redone(nn);
  std::vector<double> ld_leaf(nleaf), ld_node(nn);
  BGP_CUDA(cudaMemcpyAsync(&bad_row, f->bad_row.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  if (nn) BGP_CUDA(cudaMemcpyAsync(status.data(), f->status.p, sizeof(int) * nn, cudaMemcpyDeviceToHost, s));
  if (nn) BGP_CUDA(cudaMemcpyAsync(redone.data(), f->redone.p, sizeof(int) * nn, cudaMemcpyDeviceToHost, s));
  if (nn) BGP_CUDA(cudaMemcpyAsync(ld_node.data(), f->node_logdet.p, sizeof(double) * nn, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaMemcpyAsync(ld_leaf.data(), f->leaf_logdet.p, sizeof(double) * nleaf, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  float ms = 0.f;
  cudaEventElapsedTime(&ms, f->ev[0], f->ev[1]);
  f->build_ms = ms;
  f->householder_nodes.assign(nlev, 0);
  for (int l = 0; l < nlev; ++l)
    for (int b = 0; b < f->levels[l].nn; ++b) f->householder_nodes[l] += redone[f->levels[l].node0 + b];
  if (bad_row != no_row) {
    int li = 0;
    while (li + 1 < nleaf && f->leaves[li].start + f->leaves[li].size <= bad_row) ++li;
    const SymLeaf& lf = f->leaves[li];
    const int i = bad_row - lf.start;
    double d = 0.0;
    BGP_CUDA(cudaMemcpy(&d, dL + lf.off + (int64_t)i * lf.size + i, sizeof(double), cudaMemcpyDeviceToHost));
    set_error("the HODLR matrix is not positive definite: leaf %d (rows [%d, %d)) has the L D L^T pivot D = %g at row %d, "
              "so it has no symmetric factor", li, lf.start, lf.start + lf.size, d, bad_row);
    return BGP_ERR_LINALG;
  }
  for (int l = nlev - 1; l >= 0; --l) {  // the first failure in build order
    const SymLevelHost& L = f->levels[l];
    for (int b = 0; b < L.nn; ++b) {
      const int k = L.node0 + b;
      if (status[k] == 0) continue;
      const SymNode& d = f->nodes[k];
      if (status[k] == 1)
        set_error("the low-rank factors of node %d (rows [%d, %d), level %d) are not finite, so the HODLR matrix has no "
                  "symmetric factor", f->node_id[k], d.start, d.start + d.size, l);
      else
        set_error("the HODLR matrix is not positive definite: node %d (rows [%d, %d), level %d, rank %d) has no "
                  "symmetric factor (I + M is not positive definite)", f->node_id[k], d.start, d.start + d.size, l,
                  d.rank);
      return BGP_ERR_LINALG;
    }
  }
  double ld = 0.0;
  for (double v : ld_leaf) ld += v;
  for (double v : ld_node) ld += 2.0 * v;
  f->logdet = ld;
  *logdet_out = ld;
  return BGP_OK;
}

// Z (n x nrhs on the device, leading dimension n) <- W Z (transpose = 0) or W^T Z, in groups of 64 columns
static int sym_apply_dev(SymFactor* f, double* Z, int64_t nrhs, int transpose, cudaStream_t s) {
  const int nlev = (int)f->levels.size();
  for (int64_t c0 = 0; c0 < nrhs; c0 += 64) {
    const int nc = (int)std::min<int64_t>(64, nrhs - c0);
    double* X = Z + c0 * f->n;
    if (!transpose) {
      for (int l = 0; l < nlev; ++l) BGP_TRY(level_apply(f, f->levels[l], X, nc, 0, s));
      BGP_TRY(launch_leaf_product(f, X, nc, 0, s));
    } else {
      BGP_TRY(launch_leaf_product(f, X, nc, 1, s));
      for (int l = nlev - 1; l >= 0; --l) BGP_TRY(level_apply(f, f->levels[l], X, nc, 1, s));
    }
  }
  return BGP_OK;
}

// z: host, column-major (n x nrhs, leading dimension ldz), in place; staged through a device buffer of 64 columns
// (N x 64 doubles, 128 MiB at N = 2^18, kept on the handle), one group at a time
int sym_apply(SymFactor* f, double* z, int64_t nrhs, int64_t ldz, int transpose, cudaStream_t s) {
  const int64_t slab = 64;
  f->apply_ms = 0.0;
  for (int64_t c0 = 0; c0 < nrhs; c0 += slab) {
    const int64_t nc = std::min(slab, nrhs - c0);
    BGP_TRY(f->z.reserve((size_t)f->n * nc, s));
    BGP_CUDA(cudaMemcpy2DAsync(f->z.p, sizeof(double) * f->n, z + c0 * ldz, sizeof(double) * ldz,
                               sizeof(double) * f->n, nc, cudaMemcpyHostToDevice, s));
    BGP_CUDA(cudaEventRecord(f->ev[0], s));
    BGP_TRY(sym_apply_dev(f, f->z.p, nc, transpose, s));
    BGP_CUDA(cudaEventRecord(f->ev[1], s));
    BGP_CUDA(cudaMemcpy2DAsync(z + c0 * ldz, sizeof(double) * ldz, f->z.p, sizeof(double) * f->n,
                               sizeof(double) * f->n, nc, cudaMemcpyDeviceToHost, s));
    BGP_CUDA(cudaStreamSynchronize(s));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, f->ev[0], f->ev[1]);
    f->apply_ms += ms;
  }
  return BGP_OK;
}

// max over the nodes of max |Q_h^T Q_h - I| (test diagnostic)
int sym_orthogonality(SymFactor* f, double* out, cudaStream_t s) {
  const int nn = (int)f->nodes.size();
  BGP_TRY(f->orth.reserve(std::max(nn, 1), s));
  BGP_CUDA(cudaMemsetAsync(f->orth.p, 0, sizeof(double) * std::max(nn, 1), s));
  for (const SymLevelHost& L : f->levels) {
    if (L.r == 0) continue;
    BGP_TRY(launch_tn(f, L, f->P.p, L.ucol, L.r, s));
    sym_orth_kernel<<<L.nn, SY_THREADS, 0, s>>>(f->d_nodes.p + L.node0, f->part.p, nchunks_of(L), f->orth.p, nullptr,
                                                0.0, L.node0);
    BGP_LAUNCH_CHECK();
  }
  std::vector<double> v(std::max(nn, 1));
  BGP_CUDA(cudaMemcpyAsync(v.data(), f->orth.p, sizeof(double) * v.size(), cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  double m = 0.0;
  for (double x : v) m = std::max(m, x);
  *out = m;
  return BGP_OK;
}

int sym_householder_nodes(const SymFactor* f, int32_t* counts, int32_t cap) {
  const int nlev = (int)f->householder_nodes.size();
  for (int l = 0; l < std::min(cap, nlev); ++l) counts[l] = f->householder_nodes[l];
  return nlev;
}

void sym_timing(const SymFactor* f, double* ms2) {
  ms2[0] = f->build_ms;
  ms2[1] = f->apply_ms;
}

}  // namespace bgp
