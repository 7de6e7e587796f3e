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
// On a shard (DESIGN.md §5) the build splits at the shard cut: sym_build_local runs steps 1-3 on the shard's leaves and
// owned levels, each owned node also applying W_v^-1 to the top levels' columns on its rows; once every shard's rows of
// those columns are in place (the caller's all-gather), sym_build_top runs step 3 for the levels above the cut over all
// N rows, identically on every shard.  The apply splits the same way (apply_group's parts).
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <vector>

#include "hodlr_sym.cuh"

namespace bgp {

struct SymLevelHost {
  int r = 0, ucol = 0, vcol = 0, node0 = 0, nn = 0, max_size = 0, max_half = 0;
  int set = 1;  // 0: above the shard cut (the top panel, all N rows), 1: owned (the local panel, this shard's rows)
  int64_t q_base = 0, x_base = 0;
};

// The factor panel P in two parts, as compute()'s panel sets (DESIGN.md §3): the top part (N x rtop, leading dimension
// N) holds the columns of the levels above the shard cut, the local part (nloc x rloc, leading dimension nloc) those of
// the owned levels, addressed with global rows through a base shifted by row0.  Unsharded: no top part, row0 = 0,
// nloc = N.
struct SymFactor {
  int64_t n = 0, row0 = 0, nloc = 0;
  int cut = 0, rtop = 0, rloc = 0, max_leaf = 0;
  std::vector<SymLevelHost> levels;
  std::vector<SymNode> nodes;   // level by level, deepest level last
  std::vector<int> node_id;     // pre-order id of each entry of `nodes`
  std::vector<SymLeaf> leaves;  // ncols: the leaf's ancestor columns in the local part
  const double* dL = nullptr;   // the handle's leaf factors (valid while the factorisation is)
  double logdet_local = 0.0;    // the leaves' and the owned nodes' terms of log|K~|
  double logdet = 0.0;
  DevBuf<SymNode> d_nodes;
  DevBuf<SymLeaf> d_leaves, d_leaves_top;  // d_leaves_top: the same leaves over all rtop top columns
  DevBuf<double> P, Ptop, XY, QR, part, tbuf, ubuf, z, leaf_logdet, node_logdet, orth, acopy;
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

// the level's own part of P: its base (global rows) and leading dimension
static double* pbase(const SymFactor* f, const SymLevelHost& L) { return L.set == 0 ? f->Ptop.p : f->P.p - f->row0; }
static int64_t pld(const SymFactor* f, const SymLevelHost& L) { return L.set == 0 ? f->n : f->nloc; }

// the leaf kernels stage (max_leaf x cols) doubles: 8 columns for leaves of up to 3200 rows, one column beyond
static int leaf_cols(int max_leaf) {
  return sizeof(double) * (size_t)max_leaf * SY_LEAF_COLS <= SY_SMEM_MAX ? SY_LEAF_COLS : 1;
}

// X <- D^-1/2 L^-1 X on every leaf's rows over its leaves[].ncols columns (at most maxc)
static int launch_leaf_forward(SymFactor* f, const SymLeaf* leaves, int maxc, double* X, int64_t ldx, cudaStream_t s) {
  if (maxc == 0 || f->leaves.empty()) return BGP_OK;
  const int cols = leaf_cols(f->max_leaf), ngroups = (maxc + cols - 1) / cols;
  const dim3 grid((unsigned)(f->leaves.size() * (size_t)ngroups));
  const size_t smem = sizeof(double) * (size_t)f->max_leaf * cols;
  if (cols == SY_LEAF_COLS)
    sym_leaf_forward_kernel<SY_LEAF_COLS><<<grid, SY_THREADS, smem, s>>>(leaves, f->dL, X, ldx, f->max_leaf, ngroups);
  else
    sym_leaf_forward_kernel<1><<<grid, SY_THREADS, smem, s>>>(leaves, f->dL, X, ldx, f->max_leaf, ngroups);
  BGP_LAUNCH_CHECK();
  return BGP_OK;
}

static int launch_leaf_product(SymFactor* f, double* Z, int64_t ldz, int nc, int transpose, cudaStream_t s) {
  if (f->leaves.empty()) return BGP_OK;
  const int cols = leaf_cols(f->max_leaf), ngroups = (nc + cols - 1) / cols;
  const dim3 grid((unsigned)(f->leaves.size() * (size_t)ngroups));
  const size_t smem = sizeof(double) * (size_t)f->max_leaf * cols;
  if (cols == SY_LEAF_COLS)
    sym_leaf_product_kernel<SY_LEAF_COLS><<<grid, SY_THREADS, smem, s>>>(f->d_leaves.p, f->dL, Z, ldz, nc,
                                                                          f->max_leaf, ngroups, transpose);
  else
    sym_leaf_product_kernel<1><<<grid, SY_THREADS, smem, s>>>(f->d_leaves.p, f->dL, Z, ldz, nc, f->max_leaf, ngroups,
                                                               transpose);
  BGP_LAUNCH_CHECK();
  return BGP_OK;
}

static int nchunks_of(const SymLevelHost& L) { return std::max(1, (L.max_half + 1 + SY_TN_CHUNK - 1) / SY_TN_CHUNK); }

// partial products Q_h^T B_h of every node of level L, for columns [bcol0, bcol0 + ncols) of B (leading dimension ldb)
static int launch_tn(SymFactor* f, const SymLevelHost& L, const double* B, int64_t ldb, int bcol0, int ncols,
                     cudaStream_t s) {
  const int nch = nchunks_of(L);
  BGP_TRY(f->part.reserve((size_t)L.nn * 2 * nch * L.r * ncols, s));
  for (int b0 = 0; b0 < L.nn; b0 += SY_LEVEL_SLAB) {
    const int nb = std::min(SY_LEVEL_SLAB, L.nn - b0);
    const dim3 grid((unsigned)nch, (unsigned)(2 * nb), (unsigned)((ncols + SY_TN_TC - 1) / SY_TN_TC));
    sym_tn_kernel<<<grid, SY_THREADS, 0, s>>>(f->d_nodes.p + L.node0, pbase(f, L), pld(f, L), B, ldb, bcol0, ncols,
                                              f->part.p, nch, b0);
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
                     double* O, int64_t ldo, int ocol0, int ncols, int accumulate, cudaStream_t s) {
  const int rows = nn_rows(L.r);
  const size_t smem = sizeof(double) * rows * (size_t)(L.r + 1);
  for (int b0 = 0; b0 < L.nn; b0 += SY_LEVEL_SLAB) {
    const int nb = std::min(SY_LEVEL_SLAB, L.nn - b0);
    const dim3 grid((unsigned)((L.max_half + 1 + rows - 1) / rows), (unsigned)(2 * nb));
    sym_nn_kernel<<<grid, SY_THREADS, smem, s>>>(f->d_nodes.p + L.node0, pbase(f, L), pld(f, L), T, tstride, thalf, ldt,
                                                 O, ldo, ocol0, ncols, accumulate, rows, b0);
    BGP_LAUNCH_CHECK();
  }
  return BGP_OK;
}

// Z[:, 0:ncols] += Q_v S_op Q_v^T Z on every node of level L (op: 0 = X, 1 = X^T, 2 = Y); Z leading dimension ldz
static int level_apply(SymFactor* f, const SymLevelHost& L, double* Z, int64_t ldz, int ncols, int op, cudaStream_t s) {
  if (L.r == 0 || ncols == 0) return BGP_OK;
  BGP_TRY(launch_tn(f, L, Z, ldz, 0, ncols, s));
  const size_t tsz = (size_t)L.nn * 2 * L.r * ncols;
  BGP_TRY(f->tbuf.reserve(tsz, s));
  BGP_TRY(f->ubuf.reserve(tsz, s));
  sym_mid_kernel<<<L.nn, SY_THREADS, 0, s>>>(f->d_nodes.p + L.node0, f->part.p, nchunks_of(L), ncols, f->XY.p, op,
                                             f->tbuf.p, f->ubuf.p);
  BGP_LAUNCH_CHECK();
  return launch_nn(f, L, f->ubuf.p, (int64_t)2 * L.r * ncols, L.r, 2 * L.r, Z, ldz, 0, ncols, 1, s);
}

// Validates the tree and reserves every buffer of the build and of one 64-column apply group (with `staging`, the
// N x 64 host-apply staging too); launches nothing, so that sharded callers can agree on the outcome first.
//   lev:    per level (root first) r, ucol, vcol, node count; levels [0, cut) are above the shard cut
//   nodes:  per node (level order) start, size, half, rank, pre-order id
//   leaves: per leaf start, size, local ancestor columns, offset of its L D L^T block in dL
int sym_prepare(SymFactor* f, int64_t n, int64_t row0, int64_t nloc, int cut, int nlev, const int* lev,
                const int* nodes, int nleaf, const int64_t* leaves, int max_leaf, const double* dL, bool staging,
                cudaStream_t s) {
  set_sym_func_attrs();
  f->n = n; f->row0 = row0; f->nloc = nloc; f->cut = cut; f->max_leaf = max_leaf; f->dL = dL;
  f->levels.assign(nlev, SymLevelHost());
  f->nodes.clear(); f->node_id.clear(); f->leaves.clear();
  int64_t q_total = 0, x_total = 0;
  f->rtop = 0; f->rloc = 0;
  for (int l = 0, k = 0; l < nlev; ++l) {
    SymLevelHost& L = f->levels[l];
    L.r = lev[4 * l]; L.ucol = lev[4 * l + 1]; L.vcol = lev[4 * l + 2]; L.nn = lev[4 * l + 3];
    L.set = l < cut ? 0 : 1;
    L.node0 = (int)f->nodes.size();
    L.q_base = q_total; L.x_base = x_total;
    int& rset = L.set == 0 ? f->rtop : f->rloc;
    rset = std::max(rset, L.ucol + L.r);
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
  BGP_TRY(f->d_nodes.reserve(std::max(nn, 1), s));
  BGP_TRY(f->d_leaves.reserve(std::max(nleaf, 1), s));
  if (f->rtop) BGP_TRY(f->d_leaves_top.reserve(std::max(nleaf, 1), s));
  BGP_TRY(f->P.reserve((size_t)nloc * std::max(f->rloc, 1), s));
  if (f->rtop) BGP_TRY(f->Ptop.reserve((size_t)n * f->rtop, s));
  BGP_TRY(f->QR.reserve((size_t)std::max<int64_t>(q_total, 1), s));
  BGP_TRY(f->XY.reserve((size_t)std::max<int64_t>(x_total, 1), s));
  BGP_TRY(f->leaf_logdet.reserve(std::max(nleaf, 1), s));
  BGP_TRY(f->node_logdet.reserve(std::max(nn, 1), s));
  BGP_TRY(f->status.reserve(std::max(nn, 1), s));
  BGP_TRY(f->redone.reserve(std::max(nn, 1), s));
  BGP_TRY(f->bad_row.reserve(1, s));
  int max_r = 1;
  size_t part_need = 1, t_need = 1, copy_need = 1;
  for (const SymLevelHost& L : f->levels) {
    max_r = std::max(max_r, L.r);
    copy_need = std::max(copy_need, (size_t)pld(f, L) * L.r);
    // widest product of the level: its own columns (QR), its ancestors' (the update) or a 64-column apply group
    const size_t c = (size_t)std::max({L.r, L.ucol, L.set == 1 ? f->rtop : 0, 64});
    part_need = std::max(part_need, (size_t)L.nn * 2 * nchunks_of(L) * L.r * c);
    t_need = std::max(t_need, (size_t)L.nn * 2 * L.r * c);
  }
  BGP_TRY(f->acopy.reserve(copy_need, s));
  BGP_TRY(f->part.reserve(part_need, s));
  BGP_TRY(f->tbuf.reserve(t_need, s));
  BGP_TRY(f->ubuf.reserve(t_need, s));
  if (staging) BGP_TRY(f->z.reserve((size_t)n * 64, s));
  if (!f->ev[0]) {
    BGP_CUDA(cudaEventCreate(&f->ev[0]));
    BGP_CUDA(cudaEventCreate(&f->ev[1]));
  }
  return BGP_OK;
}

// Level l's step of the build (step 3): orthonormal bases of its nodes' own columns, the 2r x 2r steps, and W_v^-1 on
// the ancestor columns over the node's rows: [0, ucol) of the level's own part and, for an owned level, all rtop
// columns of the top part.
static int build_level(SymFactor* f, int l, bool all_householder, cudaStream_t s) {
  const SymLevelHost& L = f->levels[l];
  if (L.r == 0) return BGP_OK;
  double* const Pl = pbase(f, L);
  const int64_t ld = pld(f, L), roff = L.set == 0 ? 0 : f->row0;
  BGP_CUDA(cudaMemcpyAsync(f->acopy.p, Pl + (int64_t)L.ucol * ld + roff, sizeof(double) * ld * L.r,
                           cudaMemcpyDeviceToDevice, s));
  for (int pass = 0; pass < (all_householder ? 0 : 3); ++pass) {
    BGP_TRY(launch_tn(f, L, Pl, ld, L.ucol, L.r, s));
    sym_qr_pass_kernel<<<L.nn, SY_THREADS, sizeof(double) * L.r, s>>>(f->d_nodes.p + L.node0, f->part.p, nchunks_of(L),
                                                                      f->QR.p, pass, f->status.p, L.node0);
    BGP_LAUNCH_CHECK();
    const int64_t rr = (int64_t)L.r * L.r;
    BGP_TRY(launch_nn(f, L, f->QR.p + L.q_base + 2 * rr, 6 * rr, rr, L.r, Pl, ld, L.ucol, L.r, 0, s));
  }
  BGP_TRY(launch_tn(f, L, Pl, ld, L.ucol, L.r, s));
  // (all_householder: a bar below every |Q^T Q - I| marks every node of nonzero rank)
  sym_orth_kernel<<<L.nn, SY_THREADS, 0, s>>>(f->d_nodes.p + L.node0, f->part.p, nchunks_of(L), nullptr, f->status.p,
                                              all_householder ? -1.0 : SY_ORTH_BAR, L.node0);
  BGP_LAUNCH_CHECK();
  // (the copy's column q sits at acopy + q ld over the part's rows: shift the base so that the kernel's column ucol + q,
  //  global row i, lands there)
  sym_householder_kernel<<<L.nn, SY_THREADS, sizeof(double) * L.r, s>>>(
      f->d_nodes.p + L.node0, f->acopy.p - (int64_t)L.ucol * ld - roff, ld, Pl, ld, f->QR.p, f->status.p, f->redone.p,
      L.node0);
  BGP_LAUNCH_CHECK();
  sym_node_kernel<<<L.nn, SY_THREADS, 0, s>>>(f->d_nodes.p + L.node0, f->QR.p, f->XY.p, f->node_logdet.p, f->status.p,
                                              L.node0);
  BGP_LAUNCH_CHECK();
  auto inverse_update = [&](double* B, int64_t ldb, int ncols) -> int {  // W_v^-1 on columns [0, ncols) of B
    BGP_TRY(launch_tn(f, L, B, ldb, 0, ncols, s));
    const size_t tsz = (size_t)L.nn * 2 * L.r * ncols;
    BGP_TRY(f->tbuf.reserve(tsz, s));
    BGP_TRY(f->ubuf.reserve(tsz, s));
    sym_mid_kernel<<<L.nn, SY_THREADS, 0, s>>>(f->d_nodes.p + L.node0, f->part.p, nchunks_of(L), ncols, f->XY.p, 2,
                                               f->tbuf.p, f->ubuf.p);
    BGP_LAUNCH_CHECK();
    return launch_nn(f, L, f->ubuf.p, (int64_t)2 * L.r * ncols, L.r, 2 * L.r, B, ldb, 0, ncols, 1, s);
  };
  if (L.ucol > 0) BGP_TRY(inverse_update(Pl, ld, L.ucol));
  if (L.set == 1 && f->rtop > 0) BGP_TRY(inverse_update(f->Ptop.p, f->n, f->rtop));
  return BGP_OK;
}

// The statuses, Householder counts and log-determinant terms of levels [l0, l1) (and with `leaves`, of the leaves)
// after the stream has drained: BGP_ERR_LINALG naming the first failure in build order, else *ld gets the leaves'
// terms (with `leaves`) plus twice the nodes' sums, in level order.
static int collect(SymFactor* f, int l0, int l1, bool leaves, cudaStream_t s, double* ld_out) {
  const int nn = (int)f->nodes.size(), nleaf = (int)f->leaves.size(), nlev = (int)f->levels.size();
  const int no_row = 0x7fffffff;
  int bad_row = no_row;
  std::vector<int> status(nn), redone(nn);
  std::vector<double> ld_leaf(nleaf), ld_node(nn);
  if (leaves) BGP_CUDA(cudaMemcpyAsync(&bad_row, f->bad_row.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  if (nn) BGP_CUDA(cudaMemcpyAsync(status.data(), f->status.p, sizeof(int) * nn, cudaMemcpyDeviceToHost, s));
  if (nn) BGP_CUDA(cudaMemcpyAsync(redone.data(), f->redone.p, sizeof(int) * nn, cudaMemcpyDeviceToHost, s));
  if (nn) BGP_CUDA(cudaMemcpyAsync(ld_node.data(), f->node_logdet.p, sizeof(double) * nn, cudaMemcpyDeviceToHost, s));
  if (leaves && nleaf)
    BGP_CUDA(cudaMemcpyAsync(ld_leaf.data(), f->leaf_logdet.p, sizeof(double) * nleaf, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  f->householder_nodes.resize(nlev, 0);
  for (int l = l0; l < l1; ++l) {
    f->householder_nodes[l] = 0;
    for (int b = 0; b < f->levels[l].nn; ++b) f->householder_nodes[l] += redone[f->levels[l].node0 + b];
  }
  if (bad_row != no_row) {
    int li = 0;
    while (li + 1 < nleaf && f->leaves[li].start + f->leaves[li].size <= bad_row) ++li;
    const SymLeaf& lf = f->leaves[li];
    const int i = bad_row - lf.start;
    double d = 0.0;
    BGP_CUDA(cudaMemcpy(&d, f->dL + lf.off + (int64_t)i * lf.size + i, sizeof(double), cudaMemcpyDeviceToHost));
    set_error("the HODLR matrix is not positive definite: leaf %d (rows [%d, %d)) has the L D L^T pivot D = %g at row %d, "
              "so it has no symmetric factor", li, lf.start, lf.start + lf.size, d, bad_row);
    return BGP_ERR_LINALG;
  }
  for (int l = l1 - 1; l >= l0; --l) {  // the first failure in build order
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
  const int k0 = l0 < nlev ? f->levels[l0].node0 : nn, k1 = l1 < nlev ? f->levels[l1].node0 : nn;
  for (int k = k0; k < k1; ++k) ld += 2.0 * ld_node[k];
  *ld_out = ld;
  return BGP_OK;
}

// Steps 1-3 on this shard's part (sym_prepare first): the used V columns into both parts of P (the top levels' V,
// `vtop`, spans all N rows with leading dimension N; the owned levels' `vloc` is addressed with global rows), the
// leaves over the local ancestor columns and over all top columns on their rows, and the owned levels, deepest first.
// The top part then holds, on this shard's rows, what the top levels need from it.  Unsharded, this is the whole build.
int sym_build_local(SymFactor* f, const double* vtop, const double* vloc, int64_t ldvloc, cudaStream_t s) {
  const int nn = (int)f->nodes.size(), nleaf = (int)f->leaves.size(), nlev = (int)f->levels.size();
  // BGP_SYM_QR=householder (diagnostic): every node through the Householder QR, none through CholeskyQR3
  const char* qr_env = getenv("BGP_SYM_QR");
  const bool all_householder = qr_env && !strcmp(qr_env, "householder");
  if (nn) BGP_CUDA(cudaMemcpyAsync(f->d_nodes.p, f->nodes.data(), sizeof(SymNode) * nn, cudaMemcpyHostToDevice, s));
  BGP_CUDA(cudaMemcpyAsync(f->d_leaves.p, f->leaves.data(), sizeof(SymLeaf) * nleaf, cudaMemcpyHostToDevice, s));
  std::vector<SymLeaf> top_leaves(f->leaves);
  if (f->rtop) {
    for (SymLeaf& lf : top_leaves) lf.ncols = f->rtop;
    BGP_CUDA(cudaMemcpyAsync(f->d_leaves_top.p, top_leaves.data(), sizeof(SymLeaf) * nleaf, cudaMemcpyHostToDevice, s));
  }
  BGP_CUDA(cudaMemsetAsync(f->status.p, 0, sizeof(int) * std::max(nn, 1), s));
  BGP_CUDA(cudaMemsetAsync(f->redone.p, 0, sizeof(int) * std::max(nn, 1), s));
  BGP_CUDA(cudaMemsetAsync(f->node_logdet.p, 0, sizeof(double) * std::max(nn, 1), s));  // levels of rank 0 add nothing
  const int no_row = 0x7fffffff;
  BGP_CUDA(cudaMemcpyAsync(f->bad_row.p, &no_row, sizeof(int), cudaMemcpyHostToDevice, s));

  BGP_CUDA(cudaEventRecord(f->ev[0], s));
  // 1. P <- the used V columns
  for (const SymLevelHost& L : f->levels) {
    if (L.r == 0) continue;
    const double* V = L.set == 0 ? vtop : vloc;
    const int64_t ldv = L.set == 0 ? f->n : ldvloc;
    for (int b0 = 0; b0 < L.nn; b0 += SY_LEVEL_SLAB) {
      const int nb = std::min(SY_LEVEL_SLAB, L.nn - b0);
      sym_copy_kernel<<<dim3((unsigned)((L.max_size + SY_THREADS - 1) / SY_THREADS), (unsigned)nb), SY_THREADS, 0, s>>>(
          f->d_nodes.p + L.node0 + b0, V, ldv, L.vcol, pbase(f, L), pld(f, L));
      BGP_LAUNCH_CHECK();
    }
  }
  // 2. leaves: D > 0, log|D|, P <- D^-1/2 L^-1 P
  if (nleaf) {
    sym_leaf_check_kernel<<<nleaf, SY_THREADS, 0, s>>>(f->d_leaves.p, f->dL, f->leaf_logdet.p, f->bad_row.p);
    BGP_LAUNCH_CHECK();
  }
  int maxc = 0;
  for (const SymLeaf& lf : f->leaves) maxc = std::max(maxc, lf.ncols);
  BGP_TRY(launch_leaf_forward(f, f->d_leaves.p, maxc, f->P.p - f->row0, f->nloc, s));
  if (f->rtop) BGP_TRY(launch_leaf_forward(f, f->d_leaves_top.p, f->rtop, f->Ptop.p, f->n, s));
  // 3. owned levels, deepest first
  for (int l = nlev - 1; l >= f->cut; --l) BGP_TRY(build_level(f, l, all_householder, s));
  BGP_CUDA(cudaEventRecord(f->ev[1], s));
  BGP_CUDA(cudaEventSynchronize(f->ev[1]));
  float ms = 0.f;
  cudaEventElapsedTime(&ms, f->ev[0], f->ev[1]);
  f->build_ms = ms;
  f->householder_nodes.assign(nlev, 0);
  return collect(f, std::min(f->cut, nlev), nlev, true, s, &f->logdet_local);
}

// The top part of P after every shard's rows of it are in place: the levels above the cut over all N rows (the same
// launches on the same data on every shard).  *logdet_out = the local terms plus, with add_top, the top nodes' terms.
int sym_build_top(SymFactor* f, int add_top, cudaStream_t s, double* logdet_out) {
  const int nlev = (int)f->levels.size(), cut = std::min(f->cut, nlev);
  const char* qr_env = getenv("BGP_SYM_QR");
  const bool all_householder = qr_env && !strcmp(qr_env, "householder");
  BGP_CUDA(cudaEventRecord(f->ev[0], s));
  for (int l = cut - 1; l >= 0; --l) BGP_TRY(build_level(f, l, all_householder, s));
  BGP_CUDA(cudaEventRecord(f->ev[1], s));
  double ld_top = 0.0;
  BGP_TRY(collect(f, 0, cut, false, s, &ld_top));
  float ms = 0.f;
  cudaEventElapsedTime(&ms, f->ev[0], f->ev[1]);
  f->build_ms += ms;
  f->logdet = cut == 0 ? f->logdet_local : f->logdet_local + (add_top ? ld_top : 0.0);
  *logdet_out = f->logdet;
  return BGP_OK;
}

// the top part of P (N x cols, leading dimension N), for the exchange of this shard's rows
double* sym_top_panel(SymFactor* f, int64_t* cols) {
  *cols = f->rtop;
  return f->Ptop.p;
}

// One group of nc <= 64 columns of Z (leading dimension ldz): W Z (transpose = 0) or W^T Z, part 0 = all of it, 1 = the
// owned levels and the leaves (this shard's rows only), 2 = the levels above the cut (all rows).  W runs the top levels
// first, W^T last.
static int apply_group(SymFactor* f, double* X, int64_t ldz, int nc, int transpose, int part, cudaStream_t s) {
  const int nlev = (int)f->levels.size(), cut = std::min(f->cut, nlev);
  if (!transpose) {
    if (part != 1)
      for (int l = 0; l < cut; ++l) BGP_TRY(level_apply(f, f->levels[l], X, ldz, nc, 0, s));
    if (part != 2) {
      for (int l = cut; l < nlev; ++l) BGP_TRY(level_apply(f, f->levels[l], X, ldz, nc, 0, s));
      BGP_TRY(launch_leaf_product(f, X, ldz, nc, 0, s));
    }
  } else {
    if (part != 2) {
      BGP_TRY(launch_leaf_product(f, X, ldz, nc, 1, s));
      for (int l = nlev - 1; l >= cut; --l) BGP_TRY(level_apply(f, f->levels[l], X, ldz, nc, 1, s));
    }
    if (part != 1)
      for (int l = cut - 1; l >= 0; --l) BGP_TRY(level_apply(f, f->levels[l], X, ldz, nc, 1, s));
  }
  return BGP_OK;
}

// Z (n x nrhs on the device, leading dimension ldz) <- part `part` of W Z or W^T Z, in groups of 64 columns
int sym_apply_dev(SymFactor* f, double* Z, int64_t ldz, int64_t nrhs, int transpose, int part, cudaStream_t s) {
  for (int64_t c0 = 0; c0 < nrhs; c0 += 64)
    BGP_TRY(apply_group(f, Z + c0 * ldz, ldz, (int)std::min<int64_t>(64, nrhs - c0), transpose, part, s));
  return BGP_OK;
}

// z: host, column-major (n x nrhs, leading dimension ldz), in place; staged through a device buffer of 64 columns
// (N x 64 doubles, 128 MiB at N = 2^18, kept on the handle), one group at a time.  With `exchange` (a sharded factor
// with a communicator) each group's own rows are all-gathered between the local and the top part.
int sym_apply(SymFactor* f, double* z, int64_t nrhs, int64_t ldz, int transpose, cudaStream_t s,
              const std::function<int(double*, int)>& exchange) {
  const int64_t slab = 64;
  f->apply_ms = 0.0;
  for (int64_t c0 = 0; c0 < nrhs; c0 += slab) {
    const int64_t nc = std::min(slab, nrhs - c0);
    BGP_TRY(f->z.reserve((size_t)f->n * nc, s));
    BGP_CUDA(cudaMemcpy2DAsync(f->z.p, sizeof(double) * f->n, z + c0 * ldz, sizeof(double) * ldz,
                               sizeof(double) * f->n, nc, cudaMemcpyHostToDevice, s));
    BGP_CUDA(cudaEventRecord(f->ev[0], s));
    if (!exchange) {
      BGP_TRY(apply_group(f, f->z.p, f->n, (int)nc, transpose, 0, s));
    } else if (!transpose) {
      BGP_TRY(apply_group(f, f->z.p, f->n, (int)nc, 0, 2, s));
      BGP_TRY(apply_group(f, f->z.p, f->n, (int)nc, 0, 1, s));
      BGP_TRY(exchange(f->z.p, (int)nc));
    } else {
      BGP_TRY(apply_group(f, f->z.p, f->n, (int)nc, 1, 1, s));
      BGP_TRY(exchange(f->z.p, (int)nc));
      BGP_TRY(apply_group(f, f->z.p, f->n, (int)nc, 1, 2, s));
    }
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
    BGP_TRY(launch_tn(f, L, pbase(f, L), pld(f, L), L.ucol, L.r, s));
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
