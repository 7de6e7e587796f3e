// hodlr.cu — host orchestration + C ABI of the HODLR solver (replaces src/george/solvers/_hodlr.cpp:36-204 and
// the hodlr::Node recursion of src/george/include/george/hodlr.h).
//
// Pipeline of one compute() (all on the device; the host only builds the O(#nodes) index structure):
//   tree geometry (host, bit-exact with hodlr.h:48-61)
//   -> [stream A] leaf build + LDL^T (K4)      [stream B] ACA of every internal node (K5)
//   -> ranks back to the host (one small D2H), per-level common ranks, panel finalisation
//   -> leaf solves applied to all ancestor columns, then per level bottom-up: gram (K6a) -> LU/solve (K6b) -> update (K6c)
//   -> log-det = sum of leaf and node log-dets.
// solve(): the same three kernels with the right-hand side as target (K7).
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <vector>

#include "common.cuh"
#include "hodlr_kernels.cuh"
#include "hodlr_lu.cuh"
#include "hodlr_aca2.cuh"
#include "hodlr_leaf.cuh"
#include "linalg.cuh"
#include "kernel_eval.cuh"

namespace bgp {
int upload_program(const DevProgram& P, DevBuf<DevProgram>& buf, cudaStream_t s);
int kmat_grad_contract_launch(const DevProgram* dprog, int nd, int np, const unsigned* which_dev, const double* x,
                              int64_t n, const double* M, int64_t ldm, const double* alpha, double ca, double cm,
                              double* g_dev, double* diag_dev, DevBuf<double>& scratch, cudaStream_t s);
int fill_identity_launch(double* A, int64_t n, cudaStream_t s);
int loo_weights_launch(const double* alpha, const double* d, int64_t n, double* q, double* c, cudaStream_t s);
int scale_rows_launch(double* X, int64_t n, int64_t ncols, int64_t ldx, const double* w, bool sqrt_w, cudaStream_t s);
int slab_diag_launch(const double* W, int64_t ldw, int64_t j0, int64_t nc, double* d, cudaStream_t s);
int loo_check_diag(const double* d, int64_t n);
int64_t grad_slab_partial_size(int64_t n, int64_t c, int np);
int64_t grad_slab_tile_size(int64_t n, int np);
int kmat_grad_slab_launch(const DevProgram* dprog, int nd, int np, const unsigned* which_dev, const double* x, int64_t n,
                          const double* W, int64_t j0, int64_t nc, int64_t jlo, int64_t jhi, const double* u,
                          const double* v, double* partial, double* tile_part, double* diag_dev, cudaStream_t s);
int kmat_grad_slab_finish(int np, int64_t jlo, int64_t jhi, const double* tile_part, double* g_dev, cudaStream_t s);
int64_t grad_slab_x_partial_size(int64_t n, int64_t c, int nd);
int kmat_grad_x_slab_launch(const DevProgram* dprog, int shape, int nd, int np, const unsigned* which_dev,
                            const double* x, int64_t n, const double* W, int64_t j0, int64_t nc, int64_t jlo,
                            int64_t jhi, const double* alpha, double* partial, double* tile_part, double* xpart,
                            double* diag_dev, double* dx_dev, cudaStream_t s);
int grad_x_resident_launch(const DevProgram& P, const DevProgram* dprog, const double* x, int64_t n, double* Kinv,
                           const double* alpha, double* dx_dev, DevBuf<double>& scratch, cudaStream_t s);
int kmat_symmetric_launch_auto(const DevProgram& P, const DevProgram* dprog, const double* x, int64_t n,
                               const double* diag_add, double* out, int64_t ld, cudaStream_t s);
int kmat_general_launch_auto(const DevProgram& P, const DevProgram* dprog, const double* x1, int64_t n1, const double* x2,
                             int64_t n2, double* out, int64_t ld, cudaStream_t s);
int kmat_diagonal_launch(const DevProgram* dprog, const double* x1, const double* x2, int64_t n, double* out,
                         cudaStream_t s, int members = 1, int64_t ostride = 0);
int64_t predict_chunk_cols(int64_t n, int64_t multiple);
int64_t predict_var_partial_size(int64_t n, int64_t c);
int predict_var_launch(const double* B, int64_t ldb, const double* W, int64_t ldw, int64_t n, int64_t c,
                       const double* kdiag, double* var, DevBuf<double>& scratch, cudaStream_t s);
int kmat_x1_grad_matvec_launch(const DevProgram& P, const DevProgram* dprog, const double* x1, int64_t n1,
                               const double* x2, int64_t n2, const double* V, int64_t ldv, double scale, int add_prior,
                               double* out, DevBuf<double>& scratch, cudaStream_t s);
int64_t x1_grad_partial_size(int64_t n1, int64_t n2, int nd);
void predict_gemm_plan(int64_t m, int64_t nn, int64_t K, int64_t* nsplit_out, int64_t* klen_out);
int predict_gemm_sub(const double* A, int64_t lda, const double* B, int64_t ldb, int64_t m, int64_t nn, int64_t K,
                     bool lower, double* C, int64_t ldc, DevBuf<double>& slices, DevBuf<GemmDesc>& descs, cudaStream_t s);
bool comm_ready();
int comm_rank();
int comm_world();
int comm_allreduce_sum_f64(double* buf, size_t count, cudaStream_t s);
int comm_allgather_f64(const double* send, double* recv, size_t count, cudaStream_t s);
struct SymFactor;  // hodlr_sym.cu: the symmetric factor K~ = W W^T
SymFactor* sym_create();
void sym_destroy(SymFactor* f);
int sym_prepare(SymFactor* f, int64_t n, int64_t row0, int64_t nloc, int cut, int nlev, const int* lev,
                const int* nodes, int nleaf, const int64_t* leaves, int max_leaf, const double* dL, bool staging,
                cudaStream_t s);
int sym_build_local(SymFactor* f, const double* vtop, const double* vloc, int64_t ldvloc, cudaStream_t s);
int sym_build_top(SymFactor* f, int add_top, cudaStream_t s, double* logdet_out);
double* sym_top_panel(SymFactor* f, int64_t* cols);
int sym_apply_dev(SymFactor* f, double* Z, int64_t ldz, int64_t nrhs, int transpose, int part, cudaStream_t s);
int sym_apply(SymFactor* f, double* z, int64_t nrhs, int64_t ldz, int transpose, cudaStream_t s,
              const std::function<int(double*, int)>& exchange);
int sym_orthogonality(SymFactor* f, double* out, cudaStream_t s);
void sym_timing(const SymFactor* f, double* ms2);
int sym_householder_nodes(const SymFactor* f, int32_t* counts, int32_t cap);
}
using namespace bgp;

struct HNode {
  int start, size, half, is_leaf, parent, dir, depth;
  int slot;        // index within its level (internal) or within the leaf list
  int rank = 0, draws = 0, fallback = 0;
  int owned = 1;   // sharding: this process factors the node locally
  int top = 0;     // sharding: node above the shard cut (finished after the exchange)
};

// Factor panels (DESIGN.md §3).  A level owned by one shard only ever touches that shard's rows, so its panels hold
// nloc rows (leading dimension nloc) and are addressed with GLOBAL row indices through a base pointer shifted by the
// shard's first row; the levels above the shard cut span all N rows.  Single-GPU runs have only the "local" set (all rows).
struct PanelSet {
  DevBuf<double> V, U;
  int64_t ld = 0, row_off = 0;
  int vcols = 0, ucols = 0;
  double* vbase() const { return V.p - row_off; }
  double* ubase() const { return U.p - row_off; }
};

struct LevelInfo {
  std::vector<int> nodes;  // pre-order ids of the internal nodes at this depth handled here
  int set = 1;             // 0: level above the shard cut (panel set `top`), 1: owned level (panel set `loc`)
  int cap = 0, max_cap = 0, vcol = 0, r = 0, ucol = 0;  // vcol / ucol: first column of the level in ITS panel set
  int max_half = 0, grow = 0;
  int desc_off = 0;  // offset of this level's NodeDesc block
};

struct AcaGraphKey {  // everything the captured ACA loop depends on
  A2Args a;
  int nn, ncc, nrc, shape, grid;
};

struct bgp_hodlr {
  cudaStream_t sA = nullptr, sB = nullptr;
  cudaEvent_t ev[8] = {nullptr};
  int64_t n = 0;
  int ndim = 0;
  bgp_hodlr_opts_t opts;
  bool computed = false;
  double log_det = 0.0;
  DevProgram prog;

  std::vector<HNode> nodes;  // pre-order
  std::vector<int> leaves;   // pre-order ids
  std::vector<LevelInfo> levels;
  std::vector<int> piv_off;  // per internal node (by pre-order id) offset into pivot arrays, -1 for leaves
  std::vector<int> h_piv_rows, h_piv_cols;
  int max_leaf = 0, rtot = 0, vcols = 0, cut_depth = 0;
  int64_t row0 = 0, nloc = 0;
  std::vector<int64_t> shard_row0, shard_rows;
  bool top_pending = false;  // sharded compute without a communicator done, the host has not called finish_top yet

  DevBuf<DevProgram> d_prog;
  DevBuf<double> d_x, d_yerr, d_diag, d_L, d_leaf_logdet, d_node_logdet, d_S, d_W, d_scalar, d_rhs;
  PanelSet top, loc;
  const PanelSet& pset(const LevelInfo& L) const { return L.set == 0 ? top : loc; }
  DevBuf<double> d_inv, d_gscratch;          // grad_terms: K^-1 (n x n) and the contraction partials
  DevBuf<double> d_xsend, d_xrecv;           // sharded runs: pack / all-gather staging
  DevBuf<unsigned> d_which;
  LuWorkspace lu_ws;                         // big-rank Woodbury step (hodlr_lu.cuh)
  DevBuf<GemmDesc> d_gram_desc, d_upd_desc;
  std::vector<NodeDesc> h_nodes;             // host copy of d_nodes
  std::vector<int> cap_hint;                 // per-level ACA capacities the previous compute() ended with
  int64_t cap_hint_n = -1;
  int cap_hint_min_size = -1;
  DevBuf<LeafDesc> d_leaves;
  DevBuf<AcaDesc> d_aca;
  DevBuf<AcaOut> d_aca_out;
  DevBuf<NodeDesc> d_nodes;
  DevBuf<PanelTile> d_ptiles;                // finalize_panels_kernel's row tiles (top set first)
  int small_limit = SS_MAX_N;                // 2r above which a level takes launch_level_big (BGP_SMALL_RANK_LIMIT)
  bool leaf_cols_wide = false;               // BGP_LEAF_COLS=32
  DevBuf<int> d_idx, d_piv_rows, d_piv_cols, d_ticket, d_chain_done, d_ncols_by_depth;
  DevBuf<uint32_t> d_chain_state;
  DevBuf<A2Node> d_a2nodes;
  DevBuf<A2State> d_a2states;
  DevBuf<MT19937> d_a2rngs;
  DevBuf<A2EPart> d_epart;
  DevBuf<int> d_cand, d_cand_k, d_cand_words, d_cand_L, d_cand_next, d_cand_live, d_cchunk_node, d_rchunk_node, d_nactive;
  DevBuf<double> d_node_box;
  DevBuf<double2> d_cand_xu, d_gbox, d_cbox;
  DevBuf<unsigned long long> d_cmax, d_stats;
  DevBuf<int4> d_work;
  DevBuf<int> d_work_count, d_iter;
  AcaGraphKey aca_key;
  cudaGraph_t aca_graph = nullptr;
  cudaGraphExec_t aca_exec = nullptr;
  cudaStream_t sC = nullptr;  // capture stream
  bool profile = false;
  std::vector<cudaEvent_t> prof_events;
  double prof[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};  // see bgp_hodlr_last_aca_profile
  uint64_t draw_paths[4] = {0, 0, 0, 0};  // see bgp_hodlr_last_draw_paths
  uint64_t eval_units[2] = {0, 0};  // see bgp_hodlr_last_eval_units
  DevBuf<double> d_vpart, d_upart, d_vmax;
  int aca_iters = 0;
  size_t w_cap = 0;

  double t_ms[5] = {0, 0, 0, 0, 0};
  double grad_t[4] = {0, 0, 0, 0};  // see bgp_hodlr_last_grad_timing
  double work[6] = {0, 0, 0, 0, 0, 0};

  SymFactor* sym = nullptr;  // the symmetric factor, built on first use after a compute() (bgp_hodlr_sym_factor)
  bool sym_current = false;  // sym belongs to the current factorisation
  int sym_stage = 0;         // host-exchange build: 0 none, 1 local part built (finish pending), -1 local part failed
  double sym_log_det = 0.0;
};

static int ensure_streams(bgp_hodlr* h) {
  if (!h->sA) {
    BGP_CUDA(cudaStreamCreateWithFlags(&h->sA, cudaStreamNonBlocking));
    BGP_CUDA(cudaStreamCreateWithFlags(&h->sB, cudaStreamNonBlocking));
    for (int i = 0; i < 8; ++i) BGP_CUDA(cudaEventCreate(&h->ev[i]));
  }
  return BGP_OK;
}

// hodlr.h:29-66: pre-order construction; a node splits iff size/2 >= min_size.
static void build_tree(bgp_hodlr* h, int start, int size, int dir, int parent, int depth) {
  HNode nd;
  nd.start = start; nd.size = size; nd.half = size / 2; nd.dir = dir; nd.parent = parent; nd.depth = depth;
  nd.is_leaf = !(nd.half >= h->opts.min_size);
  nd.slot = 0;
  const int id = (int)h->nodes.size();
  h->nodes.push_back(nd);
  if (!nd.is_leaf) {
    build_tree(h, start, nd.half, 0, id, depth + 1);
    build_tree(h, start + nd.half, size - nd.half, 1, id, depth + 1);
  }
}

static int hodlr_solve_dev(bgp_hodlr* h, double* b, int64_t nrhs, int64_t ldb, cudaStream_t s, int part,
                           int64_t eye_row0 = -1);
static int hodlr_exchange_finish(bgp_hodlr* h);

// A sharded factorisation exchanges rows through the library's communicator when it spans exactly the shards and this
// process is the handle's shard; otherwise the host runs the exchange (export/import_top, solve_local/top_dev).
static bool host_exchange(const bgp_hodlr* h) {
  return h->opts.shard_count > 1 &&
         !(comm_ready() && comm_world() == h->opts.shard_count && comm_rank() == h->opts.shard_rank);
}

// The full solves need every shard's rows: on a host-exchange shard they would apply the top levels to a vector whose
// other rows were never solved.
static int reject_host_exchange(const bgp_hodlr* h, const char* what) {
  if (!host_exchange(h)) return BGP_OK;
  set_error("%s is not available on a host-exchange shard (shard %d of %d without a matching communicator): use "
            "bgp_hodlr_solve_local_dev / bgp_hodlr_solve_top_dev", what, h->opts.shard_rank, h->opts.shard_count);
  return BGP_ERR_INVALID;
}
static int hodlr_finish_top_impl(bgp_hodlr* h, bool allreduce);

// The leaf solve stages a (max_leaf x cols) column group in shared memory: leaves of up to 3200 rows take the default
// 8 columns, larger ones (a tree whose root is one leaf, N < 2 min_size) the widest of 4, 2, 1 that fits.
constexpr size_t LS_SMEM_MAX = 200 * 1024;
constexpr int LS_MAX_LEAF = (int)(LS_SMEM_MAX / sizeof(double));  // 25600 rows: one column still fits

static bool leaf_solve_fits(int max_leaf, int cols) { return sizeof(double) * (size_t)max_leaf * cols <= LS_SMEM_MAX; }
// the group plus the kernel's diagonal blocks: at most 225 KB (LS_COLS_WIDE), within the 227 KB a CTA may opt into
static int ls_smem_limit(int cols) { return (int)(LS_SMEM_MAX + ls_smem_bytes(0, cols)); }

// cudaFuncSetAttribute applies to the current device: the sweep kernels that take more than the default 48 KB of dynamic
// shared memory get their limits once per device, not at every level of every call.
static void set_sweep_func_attrs() {
  static std::atomic<uint64_t> done{0};
  int dev = 0;
  cudaGetDevice(&dev);
  const uint64_t bit = dev < 64 ? (1ull << dev) : 0;
  if (bit && (done.load(std::memory_order_relaxed) & bit)) return;
  cudaFuncSetAttribute(leaf_solve_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, ls_smem_limit(1));
  cudaFuncSetAttribute(leaf_solve_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, ls_smem_limit(2));
  cudaFuncSetAttribute(leaf_solve_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, ls_smem_limit(4));
  cudaFuncSetAttribute(leaf_solve_kernel<LS_COLS>, cudaFuncAttributeMaxDynamicSharedMemorySize, ls_smem_limit(LS_COLS));
  cudaFuncSetAttribute(leaf_solve_kernel<LS_COLS_WIDE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                       ls_smem_limit(LS_COLS_WIDE));
  cudaFuncSetAttribute(small_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
  done.fetch_or(bit, std::memory_order_relaxed);
}

// Leaves [l0, l1) of h->leaves (l1 < 0: all of them).
template <int COLS>
static int leaf_solve_launch(bgp_hodlr* h, double* X, int64_t ldx, const int* ncols_by_depth, int ncols_fixed,
                             int max_cols, cudaStream_t s, int l0, int l1) {
  const int ngroups = (max_cols + COLS - 1) / COLS;
  const dim3 grid((unsigned)((size_t)(l1 - l0) * (size_t)ngroups));
  const size_t smem = ls_smem_bytes(h->max_leaf, COLS);
  leaf_solve_kernel<COLS><<<grid, LS_THREADS, smem, s>>>(h->d_leaves.p + l0, h->d_L.p, X, ldx, ncols_by_depth,
                                                         ncols_fixed, h->max_leaf, ngroups);
  BGP_LAUNCH_CHECK();
  return BGP_OK;
}

// l0, l1: only leaves [l0, l1) of h->leaves (a row-restricted solve, hodlr_solve_dev); l1 < 0 runs every leaf
static int launch_leaf_solve(bgp_hodlr* h, double* X, int64_t ldx, const int* ncols_by_depth, int ncols_fixed,
                             int max_cols, cudaStream_t s, int l0 = 0, int l1 = -1) {
  if (l1 < 0) l1 = (int)h->leaves.size();
  const int nl = l1 - l0;
  if (nl <= 0 || max_cols == 0) return BGP_OK;
  // only leaves handled locally are in d_leaves.  The narrowest instantiation that covers the call (1, 2, 4 or 8
  // columns; a one-column solve carries no 8-wide registers), wider calls in groups of 8.  BGP_LEAF_COLS=32 selects the
  // 32-column instantiation for calls with more than 8 columns (the up-sweep): it streams the leaf factor once per 32
  // columns instead of once per 8, but at four times the serial work per CTA it measured slower on H100 (up-sweep 3.42
  // vs 3.36 ms, Matern32 N = 262144, before the groups of a leaf were scheduled together) — kept as an experiment.
  // Leaves too large for the group in shared memory take the widest narrower one that fits.
  const int m = h->max_leaf;
  if (h->leaf_cols_wide && max_cols > LS_COLS && leaf_solve_fits(m, LS_COLS_WIDE))
    return leaf_solve_launch<LS_COLS_WIDE>(h, X, ldx, ncols_by_depth, ncols_fixed, max_cols, s, l0, l1);
  int cols = max_cols <= 1 ? 1 : max_cols <= 2 ? 2 : max_cols <= 4 ? 4 : LS_COLS;
  while (cols > 1 && !leaf_solve_fits(m, cols)) cols /= 2;
  if (!leaf_solve_fits(m, cols)) {
    set_error("leaf size %d too large for the leaf solve kernel (at most %d rows)", m, LS_MAX_LEAF);  // compute() rejects it first
    return BGP_ERR_INVALID;
  }
  switch (cols) {
    case LS_COLS: return leaf_solve_launch<LS_COLS>(h, X, ldx, ncols_by_depth, ncols_fixed, max_cols, s, l0, l1);
    case 4: return leaf_solve_launch<4>(h, X, ldx, ncols_by_depth, ncols_fixed, max_cols, s, l0, l1);
    case 2: return leaf_solve_launch<2>(h, X, ldx, ncols_by_depth, ncols_fixed, max_cols, s, l0, l1);
    default: return leaf_solve_launch<1>(h, X, ldx, ncols_by_depth, ncols_fixed, max_cols, s, l0, l1);
  }
}

// one internal level: W = V^T X (both halves), small solve, X -= U T.   factor: up-sweep (X = U panel) vs plain solve
// Two paths: ranks whose 2r x 2r Woodbury matrix fits one CTA's shared memory (the common case) run three batched
// kernels; larger ranks run the Gram / update products on DMMA and the blocked LU of hodlr_lu.cuh.
// b0, b1: only nodes [b0, b1) of L.nodes (a row-restricted solve, hodlr_solve_dev); b1 < 0 runs the whole level.  Node
// b's W block is then block b - b0.
static int launch_level_big(bgp_hodlr* h, const LevelInfo& L, double* X, int64_t ldx, int ncolsW, int own_off, int factor,
                            int col_lo, int col_hi, cudaStream_t s, int b0, int b1);

// nodes per launch of a level: the products put node * 2 + half on gridDim.y, at most 65535.  A level of 32768 nodes
// or more (N >= 2^16 min_size) runs in slabs of consecutive nodes; each node's sums are those of a single launch.
constexpr int LEVEL_SLAB = 32767;

static int launch_level(bgp_hodlr* h, const LevelInfo& L, double* X, int64_t ldx, int ncolsW, int own_off, int factor,
                        int col_lo, int col_hi, cudaStream_t s, int b0 = 0, int b1 = -1) {
  if (b1 < 0) b1 = (int)L.nodes.size();
  const int nn = b1 - b0;
  if (nn <= 0 || L.r == 0) {
    return BGP_OK;
  }
  if (nn > LEVEL_SLAB) {  // the products put node * 2 + half on gridDim.y (at most 65535): slabs of nodes, in order
    for (int c0 = b0; c0 < b1; c0 += LEVEL_SLAB)
      BGP_TRY(launch_level(h, L, X, ldx, ncolsW, own_off, factor, col_lo, col_hi, s, c0, std::min(b1, c0 + LEVEL_SLAB)));
    return BGP_OK;
  }
  const int r = L.r;
  const int64_t stride = (int64_t)2 * r * ncolsW;  // one (2r x ncolsW) block per node
  const size_t need = (size_t)nn * stride;
  if (need > h->w_cap) { set_error("internal: W workspace too small (%zu > %zu)", need, h->w_cap); return BGP_ERR_CUDA; }
  BGP_CUDA(cudaMemsetAsync(h->d_W.p, 0, sizeof(double) * need, s));
  // h->small_limit: BGP_SMALL_RANK_LIMIT=<2r> (read at compute()) lowers the switch-over so the tests can drive every
  // level through the big path
  if (2 * r > h->small_limit) return launch_level_big(h, L, X, ldx, ncolsW, own_off, factor, col_lo, col_hi, s, b0, b1);
  const NodeDesc* nd = h->d_nodes.p + L.desc_off + b0;
  const int max_nh = L.max_half + 1;
  if (r <= GTS_MAX_R) {
    dim3 grid((max_nh + GTS_ROWS - 1) / GTS_ROWS, nn * 2, (ncolsW + GTS_TC - 1) / GTS_TC);
    const double* vb = h->pset(L).vbase();
    const int64_t ldv = h->pset(L).ld;
    if (r <= 2) gram_tn_small_kernel<2><<<grid, GTS_THREADS, 0, s>>>(nd, vb, ldv, X, ldx, ncolsW, h->d_W.p, stride);
    else if (r <= 4) gram_tn_small_kernel<4><<<grid, GTS_THREADS, 0, s>>>(nd, vb, ldv, X, ldx, ncolsW, h->d_W.p, stride);
    else gram_tn_small_kernel<GTS_MAX_R><<<grid, GTS_THREADS, 0, s>>>(nd, vb, ldv, X, ldx, ncolsW, h->d_W.p, stride);
    BGP_LAUNCH_CHECK();
  } else {
    dim3 grid((max_nh + GT_CHUNK - 1) / GT_CHUNK, nn * 2, (ncolsW + GT_TC - 1) / GT_TC);
    gram_tn_kernel<<<grid, GT_THREADS, 0, s>>>(nd, h->pset(L).vbase(), h->pset(L).ld, X, ldx, ncolsW, h->d_W.p, stride);
    BGP_LAUNCH_CHECK();
  }
  {
    const size_t sbytes = sizeof(double) * (size_t)(2 * r) * (2 * r);
    small_solve_kernel<<<nn, SS_THREADS, sbytes, s>>>(nd, h->d_W.p, stride, ncolsW, own_off, factor, h->d_S.p,
                                                      h->d_node_logdet.p, L.desc_off + b0);
    BGP_LAUNCH_CHECK();
  }
  if (col_hi > col_lo) {
    dim3 grid((max_nh + UP_ROWS - 1) / UP_ROWS, nn * 2, (col_hi - col_lo + UP_TC - 1) / UP_TC);
    update_nn_kernel<<<grid, UP_THREADS, 0, s>>>(nd, h->pset(L).ubase(), h->pset(L).ld, X, ldx, col_lo, col_hi, h->d_W.p, stride, 0);
    BGP_LAUNCH_CHECK();
  }
  return BGP_OK;
}

static int launch_level_big(bgp_hodlr* h, const LevelInfo& L, double* X, int64_t ldx, int ncolsW, int own_off, int factor,
                            int col_lo, int col_hi, cudaStream_t s, int b0, int b1) {
  const int nn = b1 - b0;
  const int r = L.r, n2 = 2 * r;
  const int64_t stride = (int64_t)n2 * ncolsW;
  const int64_t ldv = h->pset(L).ld, ldu = h->pset(L).ld;
  double* W = h->d_W.p;
  constexpr int KCHUNK = 4096;  // rows per split-K slice of the Gram product
  std::vector<LuNode> lun(nn);
  std::vector<GemmDesc> gram, upd;
  int max_nh = 0;
  for (int k = 0; k < nn; ++k) {
    const int b = b0 + k;
    const HNode& nd = h->nodes[L.nodes[b]];
    const int64_t s_off = h->h_nodes[L.desc_off + b].s_off;
    lun[k].S = h->d_S.p + s_off;
    lun[k].piv = reinterpret_cast<int*>(lun[k].S + (int64_t)n2 * n2);
    lun[k].logdet = h->d_node_logdet.p + L.desc_off + b;
    double* Wn = W + (int64_t)k * stride;
    for (int hh = 0; hh < 2; ++hh) {
      const int rs = nd.start + (hh ? nd.half : 0), nh = hh ? (nd.size - nd.half) : nd.half;
      max_nh = std::max(max_nh, nh);
      for (int k0 = 0; k0 < nh; k0 += KCHUNK) {  // W_h (r x ncolsW) += V_h^T X_h
        GemmDesc g;
        g.A = h->pset(L).vbase() + (int64_t)L.vcol * ldv + rs + k0; g.lda = ldv;   // A'(q, i) = V[i + q ldv]
        g.B = X + rs + k0; g.ldb = ldx;                                   // B'(i, c) = X[i + c ldx]
        g.C = Wn + (hh ? 0 : r); g.ldc = n2;
        g.M = r; g.N = ncolsW; g.K = std::min(KCHUNK, nh - k0); g.mode = GD_ATOMIC_ADD;
        gram.push_back(g);
      }
      if (col_hi > col_lo) {  // X_h[:, col_lo:col_hi] -= U_h T_h
        GemmDesc g;
        g.A = h->pset(L).ubase() + (int64_t)L.ucol * ldu + rs; g.lda = ldu;        // A'(i, q) = U[i + q ldu]
        g.B = Wn + (hh ? r : 0) + (int64_t)col_lo * n2; g.ldb = n2;       // B'(q, c) = T[q + c 2r]
        g.C = X + rs + (int64_t)col_lo * ldx; g.ldc = ldx;
        g.M = nh; g.N = col_hi - col_lo; g.K = r; g.mode = GD_SUB;
        upd.push_back(g);
      }
    }
  }
  BGP_TRY(lu_upload(h->d_gram_desc, gram, s));
  BGP_TRY((gemm_dmma_launch<true, true>(h->d_gram_desc.p, (int)gram.size(), r, ncolsW, nullptr, s)));
  if (factor) {
    BGP_TRY(lu_upload(h->lu_ws.d_nodes, lun, s));
    dim3 grid((unsigned)std::min<int64_t>(((int64_t)n2 * n2 + 255) / 256, 4096), nn);
    lu_assemble_kernel<<<grid, 256, 0, s>>>(h->lu_ws.d_nodes.p, W, stride, r, own_off);
    BGP_LAUNCH_CHECK();
    BGP_TRY(lu_factor_batch(h->lu_ws, lun, n2, s));
    // the own columns [own_off, own_off + r) only feed S; the targets are the ancestor columns [col_lo, col_hi)
    if (col_hi > col_lo)
      BGP_TRY(lu_solve_batch(h->lu_ws, lun, n2, W + (int64_t)col_lo * n2, stride, n2, col_hi - col_lo, false, s));
  } else {
    BGP_TRY(lu_solve_batch(h->lu_ws, lun, n2, W, stride, n2, ncolsW, true, s));
  }
  if (!upd.empty()) {
    BGP_TRY(lu_upload(h->d_upd_desc, upd, s));
    BGP_TRY((gemm_dmma_launch<false, true>(h->d_upd_desc.p, (int)upd.size(), max_nh, col_hi - col_lo, nullptr, s)));
  }
  return BGP_OK;
}

// GPU-wide lock-step ACA (hodlr_aca2.cuh).  descs are in launch order; results go to houts[desc.node].
static int run_aca2(bgp_hodlr* h, const std::vector<AcaDesc>& descs, std::vector<AcaOut>& houts, cudaStream_t s) {
  const int nn = (int)descs.size();
  if (nn == 0) return BGP_OK;
  std::vector<A2Node> hn(nn);
  std::vector<int> cchunk_node, rchunk_node;
  int64_t cand_total = 0, top_cand_total = 0;
  (void)top_cand_total;
  // (the candidate scans of the nodes above the shard cut are done redundantly by every rank: with bound culling and
  //  one-candidate batches they are cheap, and a collective inside the lock-step loop would put a latency on every step)
  const bool dist_top = false;
  int capmax = 1;
  for (int i = 0; i < nn; ++i) {
    const AcaDesc& d = descs[i];
    A2Node& a = hn[i];
    a.row0 = d.row0; a.n_rows = d.n_rows; a.col0 = d.col0; a.n_cols = d.n_cols;
    a.vcol = d.vcol; a.cap = d.cap; a.pre_id = d.pre_id; a.node = d.node;
    {
      const PanelSet& ps = h->pset(h->levels[h->nodes[d.pre_id].depth]);
      a.ld = ps.ld;
      a.vbase = ps.vbase() + (int64_t)d.vcol * ps.ld;
    }
    a.idx_off = d.idx_off; a.piv_off = d.piv_off;
    a.cchunk0 = (int)cchunk_node.size(); a.n_cchunks = (d.n_cols + A2_CHUNK - 1) / A2_CHUNK;
    a.rchunk0 = (int)rchunk_node.size(); a.n_rchunks = (d.n_rows + A2_CHUNK - 1) / A2_CHUNK;
    for (int c = 0; c < a.n_cchunks; ++c) cchunk_node.push_back(i);
    for (int c = 0; c < a.n_rchunks; ++c) rchunk_node.push_back(i);
    a.bmax = std::min(A2_BMAX, d.n_rows);
    a.cand_off = cand_total; cand_total += a.bmax;
    a.is_top = (dist_top && h->nodes[d.pre_id].top) ? 1 : 0;
    if (a.is_top) top_cand_total = cand_total;
    capmax = std::max(capmax, d.cap);
  }
  const int ncc = (int)cchunk_node.size(), nrc = (int)rchunk_node.size();
  BGP_TRY(h->d_a2nodes.reserve(nn, s));
  BGP_TRY(h->d_a2states.reserve(nn, s));
  BGP_TRY(h->d_a2rngs.reserve((size_t)2 * nn, s));
  BGP_TRY(h->d_cand.reserve((size_t)cand_total, s));
  BGP_TRY(h->d_cand_k.reserve((size_t)cand_total, s));
  BGP_TRY(h->d_cand_words.reserve((size_t)cand_total, s));
  BGP_TRY(h->d_cand_L.reserve((size_t)cand_total, s));
  BGP_TRY(h->d_cand_next.reserve((size_t)cand_total, s));
  BGP_TRY(h->d_cand_live.reserve((size_t)cand_total, s));
  BGP_TRY(h->d_node_box.reserve((size_t)2 * nn, s));
  BGP_TRY(h->d_cmax.reserve((size_t)cand_total, s));
  BGP_TRY(h->d_epart.reserve((size_t)std::max(ncc, 1) * A2_NSUB, s));
  BGP_TRY(h->d_cchunk_node.reserve(ncc, s));
  BGP_TRY(h->d_rchunk_node.reserve(nrc, s));
  BGP_TRY(h->d_vpart.reserve((size_t)ncc * A2_NSUB * (capmax + 1), s));
  BGP_TRY(h->d_upart.reserve((size_t)nrc * A2_NSUB * (capmax + 1), s));
  const bool cull = shape_has_bound(h->prog.shape) && !getenv("BGP_NO_CULL");  // BGP_NO_CULL: exhaustive scan (tests compare both)
  if (cull) {
    BGP_TRY(h->d_vmax.reserve((size_t)ncc * A2_NGROUP, s));
    // a2_generate and a2_eval read vmax before a node's first factor writes it, scaled by sum_q |U(i, q)| = 0: a stale
    // NaN or Inf left in reused device memory would turn that 0 into NaN and keep candidates the bound rules out
    BGP_CUDA(cudaMemsetAsync(h->d_vmax.p, 0, sizeof(double) * ncc * A2_NGROUP, s));
    BGP_TRY(h->d_cand_xu.reserve((size_t)cand_total, s));
    BGP_TRY(h->d_gbox.reserve((size_t)ncc * A2_NGROUP, s));
    BGP_TRY(h->d_cbox.reserve((size_t)ncc, s));
  }
  BGP_TRY(h->d_nactive.reserve(2, s));
  int n_top = 0;
  for (int i = 0; i < nn; ++i) n_top += hn[i].is_top;
  BGP_TRY(h->d_stats.reserve(A2_NSTATS, s));
  int64_t work_cap = 0;
  // items per chunk: batches of up to 256 live candidates are cut into blocks of A2_CG, larger ones into A2_CG * A2_ITEM_CB
  for (int i = 0; i < nn; ++i) {
    const int big = (hn[i].bmax + A2_CG * A2_ITEM_CB - 1) / (A2_CG * A2_ITEM_CB);
    const int small = (std::min(hn[i].bmax, 256) + A2_CG - 1) / A2_CG;
    work_cap += (int64_t)hn[i].n_cchunks * std::max(big, small);
  }
  BGP_TRY(h->d_work.reserve((size_t)(2 * work_cap), s));
  BGP_TRY(h->d_work_count.reserve(4, s));  // [0..1] item counters, [2..3] consumption cursors
  BGP_TRY(h->d_iter.reserve(1, s));
  BGP_CUDA(cudaMemsetAsync(h->d_iter.p, 0, sizeof(int), s));
  BGP_CUDA(cudaMemsetAsync(h->d_work_count.p, 0, sizeof(int) * 4, s));
  BGP_CUDA(cudaMemsetAsync(h->d_stats.p, 0, sizeof(unsigned long long) * A2_NSTATS, s));
  BGP_CUDA(cudaMemcpyAsync(h->d_a2nodes.p, hn.data(), sizeof(A2Node) * nn, cudaMemcpyHostToDevice, s));
  BGP_CUDA(cudaMemcpyAsync(h->d_cchunk_node.p, cchunk_node.data(), sizeof(int) * ncc, cudaMemcpyHostToDevice, s));
  BGP_CUDA(cudaMemcpyAsync(h->d_rchunk_node.p, rchunk_node.data(), sizeof(int) * nrc, cudaMemcpyHostToDevice, s));
  BGP_CUDA(cudaMemcpyAsync(h->d_nactive.p, &nn, sizeof(int), cudaMemcpyHostToDevice, s));
  A2Args a;
  memset(&a, 0, sizeof(a));  // (the struct is also the key of the cached graph: no indeterminate padding)
  a.prog = h->d_prog.p; a.x = h->d_x.p; a.nodes = h->d_a2nodes.p; a.states = h->d_a2states.p; a.rngs = h->d_a2rngs.p; a.n_nodes = nn;
  a.tol = h->opts.tol; a.seed = (uint32_t)h->opts.seed; a.exhaust_mode = h->opts.exhaust_mode;
  a.idx_ws = h->d_idx.p; a.piv_rows = h->d_piv_rows.p; a.piv_cols = h->d_piv_cols.p;
  a.cand = h->d_cand.p; a.cand_k = h->d_cand_k.p; a.cand_words = h->d_cand_words.p; a.cmax = h->d_cmax.p; a.epart = h->d_epart.p;
  a.cchunk_node = h->d_cchunk_node.p; a.rchunk_node = h->d_rchunk_node.p; a.vpart = h->d_vpart.p; a.upart = h->d_upart.p;
  a.vmax = cull ? h->d_vmax.p : nullptr;
  a.cand_xu = cull ? h->d_cand_xu.p : nullptr;
  a.gbox = cull ? h->d_gbox.p : nullptr;
  a.cbox = cull ? h->d_cbox.p : nullptr;
  a.cand_L = h->d_cand_L.p; a.cand_next = h->d_cand_next.p; a.cand_live = h->d_cand_live.p; a.node_box = h->d_node_box.p;
  a.capmax = capmax; a.n_active = h->d_nactive.p; a.stats = h->d_stats.p;
  a.work = h->d_work.p; a.work_count = h->d_work_count.p; a.work_cursor = h->d_work_count.p + 2; a.work_cap = (int)work_cap; a.iter_ptr = h->d_iter.p;
  a.shard_rank = dist_top ? h->opts.shard_rank : 0; a.shard_count = dist_top ? h->opts.shard_count : 1;
  if (dist_top) BGP_CUDA(cudaMemcpyAsync(h->d_nactive.p + 1, &n_top, sizeof(int), cudaMemcpyHostToDevice, s));
  // (the attribute is per device / context: set it on every call, it is cheap)
  cudaFuncSetAttribute(a2_init_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(A2NodeSmem));
    cudaFuncSetAttribute(a2_decide_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(A2NodeSmem));
    cudaFuncSetAttribute(a2_finish_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(A2NodeSmem));
  a2_init_kernel<<<nn, A2_NODE_THREADS, sizeof(A2NodeSmem), s>>>(a);
  BGP_LAUNCH_CHECK();
  int active = nn, iters = 0;
  int eval_minb = A2_EVAL_MINB_DEFAULT;
  if (const char* e = getenv("BGP_EVAL_MINB")) eval_minb = atoi(e) == 3 ? 3 : 2;
  const int eval_grid = num_sms() * 6;  // persistent CTAs over the work list (2-3 resident per SM, a few rounds)
  // One lock-step iteration = eval -> decide -> vrow -> pivot -> vnorm|ucol -> finish -> tick.
  auto launch_iteration = [&](cudaStream_t st, cudaGraphConditionalHandle hnd, int use_hnd, int it_prof) -> int {
    auto mark = [&](int slot) -> int {
      if (it_prof < 0) return BGP_OK;
      const size_t need = (size_t)7 * (it_prof + 1);
      while (h->prof_events.size() < need) {
        cudaEvent_t e;
        BGP_CUDA(cudaEventCreate(&e));
        h->prof_events.push_back(e);
      }
      BGP_CUDA(cudaEventRecord(h->prof_events[(size_t)7 * it_prof + slot], st));
      return BGP_OK;
    };
    BGP_TRY(mark(0));
    a2_eval_launch(h->prog.shape, dim3(eval_grid), st, a, eval_minb);
    BGP_LAUNCH_CHECK();
    BGP_TRY(mark(1));
    a2_decide_kernel<<<nn, A2_NODE_THREADS, sizeof(A2NodeSmem), st>>>(a);
    BGP_LAUNCH_CHECK();
    BGP_TRY(mark(2));
    a2_vrow_launch(h->prog.shape, dim3(ncc, A2_NSUB), st, a);
    BGP_LAUNCH_CHECK();
    BGP_TRY(mark(3));
    a2_pivot_kernel<<<nn, 32, 0, st>>>(a);
    BGP_LAUNCH_CHECK();
    BGP_TRY(mark(4));
    a2_vnorm_ucol_launch(h->prog.shape, dim3(ncc + nrc, A2_NSUB), st, a, ncc);
    BGP_LAUNCH_CHECK();
    BGP_TRY(mark(5));
    a2_finish_kernel<<<nn, A2_NODE_THREADS, sizeof(A2NodeSmem), st>>>(a);
    BGP_LAUNCH_CHECK();
    BGP_TRY(mark(6));
    a2_tick_kernel<<<1, 1, 0, st>>>(a.iter_ptr, a.n_active, hnd, use_hnd);
    BGP_LAUNCH_CHECK();
    return BGP_OK;
  };
  const bool use_graph = !h->profile && !getenv("BGP_NO_GRAPH");
  if (use_graph) {
    // The whole loop is ONE graph launch: a WHILE node whose body is one iteration; a2_tick_kernel keeps the condition
    // up to date from the device-side count of active nodes.  The executable graph is cached: a hyper-parameter loop
    // calls compute() with the same shapes and buffers over and over.
    AcaGraphKey key;
    memset(&key, 0, sizeof(key));
    key.a = a; key.nn = nn; key.ncc = ncc; key.nrc = nrc; key.shape = h->prog.shape; key.grid = eval_grid * 4 + eval_minb;
    if (!h->aca_exec || memcmp(&key, &h->aca_key, sizeof(key)) != 0) {
      if (h->aca_exec) { cudaGraphExecDestroy(h->aca_exec); h->aca_exec = nullptr; }
      if (h->aca_graph) { cudaGraphDestroy(h->aca_graph); h->aca_graph = nullptr; }
      BGP_CUDA(cudaGraphCreate(&h->aca_graph, 0));
      cudaGraphConditionalHandle hnd;
      BGP_CUDA(cudaGraphConditionalHandleCreate(&hnd, h->aca_graph, 1, cudaGraphCondAssignDefault));
      cudaGraphNodeParams cp = {};
      cp.type = cudaGraphNodeTypeConditional;
      cp.conditional.handle = hnd;
      cp.conditional.type = cudaGraphCondTypeWhile;
      cp.conditional.size = 1;
      cudaGraphNode_t wnode;
      BGP_CUDA(cudaGraphAddNode(&wnode, h->aca_graph, nullptr, 0, &cp));
      cudaGraph_t body = cp.conditional.phGraph_out[0];
      if (!h->sC) BGP_CUDA(cudaStreamCreateWithFlags(&h->sC, cudaStreamNonBlocking));
      BGP_CUDA(cudaStreamBeginCaptureToGraph(h->sC, body, nullptr, nullptr, 0, cudaStreamCaptureModeRelaxed));
      const int rc = launch_iteration(h->sC, hnd, 1, -1);
      cudaGraph_t captured = nullptr;
      const cudaError_t ce = cudaStreamEndCapture(h->sC, &captured);
      if (rc != BGP_OK) return rc;
      if (ce != cudaSuccess) { set_error("ACA graph capture failed: %s", cudaGetErrorString(ce)); return BGP_ERR_CUDA; }
      BGP_CUDA(cudaGraphInstantiate(&h->aca_exec, h->aca_graph, 0));
      h->aca_key = key;
    }
    BGP_CUDA(cudaGraphLaunch(h->aca_exec, s));
    int it_host = 0, act2[2] = {0, 0};
    BGP_CUDA(cudaMemcpyAsync(&it_host, h->d_iter.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    BGP_CUDA(cudaMemcpyAsync(act2, h->d_nactive.p, sizeof(int) * 2, cudaMemcpyDeviceToHost, s));
    BGP_CUDA(cudaStreamSynchronize(s));
    iters = it_host;
    g_launches.fetch_add((uint64_t)7 * (uint64_t)std::max(iters - 1, 0), std::memory_order_relaxed);  // the capture counted one iteration
    if (act2[0] > 0) { set_error("ACA did not terminate"); return BGP_ERR_CUDA; }
  } else {
    while (active > 0) {
      for (int rep = 0; rep < 8; ++rep) {
        BGP_TRY(launch_iteration(s, 0, 0, h->profile ? iters : -1));
        iters++;
      }
      int act2[2] = {0, 0};
      BGP_CUDA(cudaMemcpyAsync(act2, h->d_nactive.p, sizeof(int) * 2, cudaMemcpyDeviceToHost, s));
      BGP_CUDA(cudaStreamSynchronize(s));
      active = act2[0];
      if (iters > (1 << 22)) { set_error("ACA did not terminate"); return BGP_ERR_CUDA; }
    }
  }
  h->aca_iters = iters;
  {
    unsigned long long st4[A2_NSTATS] = {0};
    BGP_CUDA(cudaMemcpyAsync(st4, h->d_stats.p, sizeof(st4), cudaMemcpyDeviceToHost, s));
    BGP_CUDA(cudaStreamSynchronize(s));
    for (int k = 0; k < 4; ++k) h->draw_paths[k] = st4[A2_PATH_REDO + k];
    h->eval_units[0] = st4[A2_UNITS_PULLED]; h->eval_units[1] = st4[A2_UNITS_LIVE];
    h->prof[1] = iters; h->prof[2] = (double)st4[0]; h->prof[3] = (double)st4[1]; h->prof[4] = (double)st4[2];
    h->prof[5] = (double)st4[3];
    if (h->profile) {
      double tot[6] = {0, 0, 0, 0, 0, 0};
      for (int i = 0; i < iters; ++i)
        for (int k = 0; k < 6; ++k) {
          float ms = 0;
          cudaEventElapsedTime(&ms, h->prof_events[(size_t)7 * i + k], h->prof_events[(size_t)7 * i + k + 1]);
          tot[k] += ms;
        }
      h->prof[0] = tot[0];
      for (int k = 0; k < 6; ++k) h->prof[6 + k] = tot[k];
    }
  }
  if (h->opts.exhaust_mode == BGP_EXHAUST_DENSE) {
    a2_dense_fill_kernel<<<dim3(nn, 64), 256, 0, s>>>(a);
    BGP_LAUNCH_CHECK();
    a2_dense_rank_kernel<<<(nn + 127) / 128, 128, 0, s>>>(a);
    BGP_LAUNCH_CHECK();
  }
  std::vector<A2State> hs(nn);
  BGP_CUDA(cudaMemcpyAsync(hs.data(), h->d_a2states.p, sizeof(A2State) * nn, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  for (int i = 0; i < nn; ++i) {
    AcaOut o;
    o.rank = hs[i].rank; o.draws = hs[i].draws; o.fallback = hs[i].fallback; o.status = hs[i].status;
    houts[descs[i].node] = o;
  }
  return BGP_OK;
}

static int hodlr_compute_dev_impl(bgp_hodlr* h, const bgp_kernel_spec_t* spec, const double* x_dev, int64_t n,
                                  int32_t ndim, const double* yerr_dev, const bgp_hodlr_opts_t* opts_in) {
  h->computed = false;
  h->sym_current = false;
  h->sym_stage = 0;
  h->top_pending = false;
  for (uint64_t& c : h->draw_paths) c = 0;  // (rng_mode = reference never runs the speculative draws)
  for (uint64_t& c : h->eval_units) c = 0;
  h->shard_row0.clear(); h->shard_rows.clear();  // only a sharded compute that cuts the tree reports ranges
  BGP_TRY(require_device());
  BGP_TRY(ensure_streams(h));
  BGP_TRY(build_dev_program(spec, &h->prog));
  if (h->prog.ndim != ndim) { set_error("dimension mismatch: kernel ndim %d, input ndim %d", h->prog.ndim, ndim); return BGP_ERR_DIM; }
  if (ndim > ACA_MAX_NDIM) { set_error("HODLR supports at most %d input dimensions", ACA_MAX_NDIM); return BGP_ERR_INVALID; }
  if (n <= 0 || n > (int64_t)0x7fffffff) { set_error("invalid number of points %lld", (long long)n); return BGP_ERR_INVALID; }
  bgp_hodlr_opts_t o;
  if (opts_in) o = *opts_in; else bgp_hodlr_default_opts(&o);
  if (o.min_size < 1) { set_error("min_size must be >= 1"); return BGP_ERR_INVALID; }
  if (o.shard_count < 1) o.shard_count = 1;
  if (o.shard_count & (o.shard_count - 1)) { set_error("shard_count must be a power of two"); return BGP_ERR_INVALID; }
  if (o.shard_rank < 0 || o.shard_rank >= o.shard_count) { set_error("invalid shard_rank"); return BGP_ERR_INVALID; }
  if (o.shard_count > 1 && o.rng_mode == BGP_RNG_REFERENCE) { set_error("rng_mode=reference serialises the tree and cannot be sharded"); return BGP_ERR_INVALID; }
  h->opts = o;
  h->n = n;
  h->ndim = ndim;
  cudaStream_t sA = h->sA, sB = h->sB;
  set_sweep_func_attrs();
  // diagnostic switches of the sweeps, fixed for this factorisation and the solves that use it
  h->small_limit = SS_MAX_N;
  if (const char* e = getenv("BGP_SMALL_RANK_LIMIT")) h->small_limit = std::min(SS_MAX_N, atoi(e));
  h->leaf_cols_wide = false;
  if (const char* e = getenv("BGP_LEAF_COLS")) h->leaf_cols_wide = atoi(e) > LS_COLS;

  // ---- tree geometry ----
  h->nodes.clear(); h->leaves.clear(); h->levels.clear();
  h->nodes.reserve(2 * (size_t)(n / std::max(1, o.min_size)) + 8);
  build_tree(h, 0, (int)n, 0, -1, 0);
  int cut = 0;
  while ((1 << cut) < o.shard_count) cut++;
  h->cut_depth = cut;
  // sharding: the sub-tree owned by this process is the depth-`cut` node number shard_rank (left-to-right);
  // if the tree is shallower than the cut, everything is "top" work done redundantly.
  int max_depth = 0;
  for (auto& nd : h->nodes) max_depth = std::max(max_depth, nd.depth);
  h->row0 = 0; h->nloc = n;
  if (o.shard_count > 1) {
    int seen = 0; bool found = false;
    for (size_t i = 0; i < h->nodes.size(); ++i) {
      HNode& nd = h->nodes[i];
      if (nd.depth == cut) {
        if (seen == o.shard_rank) { h->row0 = nd.start; h->nloc = nd.size; found = true; }
        h->shard_row0.push_back(nd.start); h->shard_rows.push_back(nd.size);
        seen++;
      }
    }
    if (!found || seen != o.shard_count) {
      h->shard_row0.clear(); h->shard_rows.clear();
      set_error("tree too shallow to shard %d ways (N=%lld, min_size=%d)", o.shard_count, (long long)n, o.min_size);
      return BGP_ERR_INVALID;
    }
    for (auto& nd : h->nodes) {
      nd.top = nd.depth < cut;
      nd.owned = !nd.top && nd.start >= h->row0 && nd.start + nd.size <= h->row0 + h->nloc;
    }
  }
  h->levels.assign(max_depth + 1, LevelInfo());
  for (size_t i = 0; i < h->nodes.size(); ++i) {
    HNode& nd = h->nodes[i];
    if (nd.is_leaf) { if (nd.owned) { nd.slot = (int)h->leaves.size(); h->leaves.push_back((int)i); } continue; }
    if (!(nd.owned || nd.top)) continue;
    LevelInfo& L = h->levels[nd.depth];
    nd.slot = (int)L.nodes.size();
    L.nodes.push_back((int)i);
    L.max_half = std::max(L.max_half, nd.size - nd.half);
  }
  while (!h->levels.empty() && h->levels.back().nodes.empty()) h->levels.pop_back();
  const int nlev = (int)h->levels.size();
  for (int l = 0; l < nlev; ++l) h->levels[l].set = (o.shard_count > 1 && l < cut) ? 0 : 1;
  h->top.ld = n; h->top.row_off = 0;
  h->loc.ld = h->nloc; h->loc.row_off = h->row0;

  // ---- capacities: start from rank_capacity (default 128) per level; levels that overflow are grown and the ACA
  //      stage is repeated (deterministic: the per-node / chained streams restart from the same seeds) ----
  const int rcap0 = o.rank_capacity > 0 ? o.rank_capacity : 128;
  for (auto& L : h->levels) {
    int mh = 0;
    for (int id : L.nodes) mh = std::max(mh, h->nodes[id].half);
    L.max_cap = std::max(1, mh);
    L.cap = std::min(rcap0, L.max_cap);
  }
  // a handle that already factored a tree of this shape starts from the capacities that run ended with (hyper-parameter
  // loops call compute() repeatedly on the same x): no repeated ACA stage in the steady state
  if (o.rank_capacity <= 0 && h->cap_hint_n == n && h->cap_hint_min_size == o.min_size && (int)h->cap_hint.size() == nlev)
    for (int l = 0; l < nlev; ++l) h->levels[l].cap = std::min(h->levels[l].max_cap, std::max(h->levels[l].cap, h->cap_hint[l]));

  // ---- inputs ----
  BGP_TRY(upload_program(h->prog, h->d_prog, sA));
  BGP_TRY(h->d_x.reserve((size_t)n * ndim, sA));
  BGP_TRY(h->d_diag.reserve((size_t)n, sA));
  if (x_dev != h->d_x.p) BGP_CUDA(cudaMemcpyAsync(h->d_x.p, x_dev, sizeof(double) * n * ndim, cudaMemcpyDeviceToDevice, sA));
  square_kernel<<<(unsigned)std::min<int64_t>((n + 255) / 256, 1184), 256, 0, sA>>>(yerr_dev, h->d_diag.p, n);
  BGP_LAUNCH_CHECK();
  BGP_CUDA(cudaEventRecord(h->ev[0], sA));  // inputs ready / timing origin

  // ---- leaves (stream A) ----
  const int nl = (int)h->leaves.size();
  std::vector<LeafDesc> hleaves(nl);
  int64_t loff = 0;
  h->max_leaf = 0;
  for (int i = 0; i < nl; ++i) {
    const HNode& nd = h->nodes[h->leaves[i]];
    hleaves[i].start = nd.start; hleaves[i].size = nd.size; hleaves[i].depth = nd.depth; hleaves[i]._pad = 0;
    hleaves[i].off = loff;
    loff += (int64_t)nd.size * nd.size;
    h->max_leaf = std::max(h->max_leaf, nd.size);
  }
  if (h->max_leaf > LS_MAX_LEAF) {
    set_error("leaf size %d too large: the leaf solve handles at most %d rows (N=%lld, min_size=%d); lower min_size",
              h->max_leaf, LS_MAX_LEAF, (long long)n, o.min_size);
    return BGP_ERR_INVALID;
  }
  BGP_TRY(h->d_leaves.reserve(std::max(nl, 1), sA));
  BGP_TRY(h->d_L.reserve((size_t)std::max<int64_t>(loff, 1), sA));
  BGP_TRY(h->d_leaf_logdet.reserve(std::max(nl, 1), sA));
  if (nl) {
    BGP_CUDA(cudaMemcpyAsync(h->d_leaves.p, hleaves.data(), sizeof(LeafDesc) * nl, cudaMemcpyHostToDevice, sA));
    // BGP_LEAF_FACTOR=generic: the CUDA-core kernel at any leaf size (tests compare the two LDL^T implementations)
    const char* lf_env = getenv("BGP_LEAF_FACTOR");
    const bool generic = lf_env && strcmp(lf_env, "generic") == 0;
    if (h->max_leaf <= LF_MAX_LEAF && !generic) {
      leaf_factor_launch(h->prog.shape, nl, h->max_leaf, sA, h->d_prog.p, h->d_x.p, h->d_diag.p, h->d_leaves.p, h->d_L.p,
                         h->d_leaf_logdet.p);
    } else {
      leaf_build_factor_kernel<<<nl, LEAF_THREADS, 0, sA>>>(h->d_prog.p, h->d_x.p, h->d_diag.p, h->d_leaves.p, h->d_L.p,
                                                            h->d_leaf_logdet.p);
    }
    BGP_LAUNCH_CHECK();
  }
  BGP_CUDA(cudaEventRecord(h->ev[1], sA));  // leaves done

  // ---- ACA (stream B, after the leaves: DESIGN.md §6) ----
  std::vector<AcaDesc> hdesc;
  std::vector<int> desc_node;  // pre-order id per descriptor
  std::vector<AcaOut> houts;
  int64_t idx_total = 0, piv_total = 0;
  int nint = 0;
  // The ACA's per-node kernels take a whole SM per CTA and can only start on an SM the leaf kernel has left, so starting
  // them beside the leaves overlaps little; after the leaves, the step measured as fast at 256-row leaves and faster at
  // 128-row ones.  The host still prepares the ACA while the leaves run.
  BGP_CUDA(cudaStreamWaitEvent(sB, h->ev[1], 0));
  for (int attempt = 0;; ++attempt) {
    int vcols_set[2] = {0, 0};
    for (auto& L : h->levels) { L.vcol = vcols_set[L.set]; vcols_set[L.set] += L.cap; }
    h->top.vcols = vcols_set[0]; h->loc.vcols = vcols_set[1];
    h->vcols = vcols_set[0] + vcols_set[1];
    hdesc.clear(); desc_node.clear();
    h->piv_off.assign(h->nodes.size(), -1);
    idx_total = 0; piv_total = 0; nint = 0;
    for (int l = 0; l < nlev; ++l) {
      for (int id : h->levels[l].nodes) {
        const HNode& nd = h->nodes[id];
        AcaDesc d;
        d.row0 = nd.start + nd.half; d.n_rows = nd.size - nd.half; d.col0 = nd.start; d.n_cols = nd.half;
        d.vcol = h->levels[l].vcol; d.cap = h->levels[l].cap; d.pre_id = id; d.node = nint;
        d.idx_off = idx_total; d.piv_off = piv_total;
        h->piv_off[id] = (int)piv_total;
        idx_total += d.n_rows; piv_total += d.cap;
        hdesc.push_back(d); desc_node.push_back(id);
        nint++;
      }
    }
    // launch order: pre-order for the chained reference stream, largest blocks first otherwise
    std::vector<int> order(nint);
    for (int i = 0; i < nint; ++i) order[i] = i;
    if (o.rng_mode == BGP_RNG_REFERENCE) std::sort(order.begin(), order.end(), [&](int a, int b) { return hdesc[a].pre_id < hdesc[b].pre_id; });
    else std::stable_sort(order.begin(), order.end(), [&](int a, int b) {
      const int ta = h->nodes[hdesc[a].pre_id].top, tb = h->nodes[hdesc[b].pre_id].top;
      if (ta != tb) return ta > tb;  // nodes above the shard cut first (contiguous candidate range for the all-reduce)
      return hdesc[a].n_rows > hdesc[b].n_rows;
    });
    std::vector<AcaDesc> hdesc_sorted(nint);
    for (int i = 0; i < nint; ++i) hdesc_sorted[i] = hdesc[order[i]];

    {
      // a capacity that no longer fits: give the old block back to the driver before asking for the larger one (the pool
      // keeps freed blocks cached, and a 2x larger request cannot reuse them: without the trim both would be resident)
      const size_t need_top = (size_t)n * std::max(h->top.vcols, 1), need_loc = (size_t)h->nloc * std::max(h->loc.vcols, 1);
      if ((h->top.V.p && h->top.V.n < need_top) || (h->loc.V.p && h->loc.V.n < need_loc)) {
        if (h->top.V.n < need_top) h->top.V.release();
        if (h->loc.V.n < need_loc) h->loc.V.release();
        h->top.U.release(); h->loc.U.release();
        BGP_CUDA(cudaStreamSynchronize(sA)); BGP_CUDA(cudaStreamSynchronize(sB));
        cudaMemPool_t pool; int dev = 0;
        cudaGetDevice(&dev);
        if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) cudaMemPoolTrimTo(pool, 0);
      }
      BGP_TRY(h->top.V.reserve(need_top, sB));
      BGP_TRY(h->loc.V.reserve(need_loc, sB));
    }
    BGP_TRY(h->d_aca.reserve(std::max(nint, 1), sB));
    BGP_TRY(h->d_aca_out.reserve(std::max(nint, 1), sB));
    BGP_TRY(h->d_idx.reserve((size_t)std::max<int64_t>(idx_total, 1), sB));
    BGP_TRY(h->d_piv_rows.reserve((size_t)std::max<int64_t>(piv_total, 1), sB));
    BGP_TRY(h->d_piv_cols.reserve((size_t)std::max<int64_t>(piv_total, 1), sB));
    BGP_TRY(h->d_ticket.reserve(1, sB));
    BGP_TRY(h->d_chain_state.reserve(640, sB));
    BGP_TRY(h->d_chain_done.reserve(std::max(nint, 1), sB));
    houts.assign(nint, AcaOut());
    if (nint && o.rng_mode != BGP_RNG_REFERENCE) {
      BGP_TRY(run_aca2(h, hdesc_sorted, houts, sB));
    } else if (nint) {
      BGP_CUDA(cudaMemcpyAsync(h->d_aca.p, hdesc_sorted.data(), sizeof(AcaDesc) * nint, cudaMemcpyHostToDevice, sB));
      BGP_CUDA(cudaMemsetAsync(h->d_ticket.p, 0, sizeof(int), sB));
      BGP_CUDA(cudaMemsetAsync(h->d_chain_done.p, 0, sizeof(int) * nint, sB));
      int maxcap = 1;
      for (auto& L : h->levels) maxcap = std::max(maxcap, L.cap);
      const size_t smem = ((sizeof(AcaShared) + 15) & ~size_t(15)) + sizeof(double) * (size_t)maxcap;
      // (the attribute is per device / context: set it on every call, it is cheap)
      cudaFuncSetAttribute(aca_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
      if (smem > 200 * 1024) { set_error("rank capacity %d too large", maxcap); return BGP_ERR_RANK_CAPACITY; }
      aca_kernel<<<nint, ACA_THREADS, smem, sB>>>(h->d_prog.p, h->d_x.p, h->d_aca.p, nint, h->loc.vbase(), h->loc.ld, o.tol, (uint32_t)o.seed,
                                                  o.rng_mode, h->d_idx.p, h->d_piv_rows.p, h->d_piv_cols.p, h->d_aca_out.p,
                                                  h->d_ticket.p, h->d_chain_state.p, h->d_chain_done.p, o.exhaust_mode);
      BGP_LAUNCH_CHECK();
      BGP_CUDA(cudaMemcpyAsync(houts.data(), h->d_aca_out.p, sizeof(AcaOut) * nint, cudaMemcpyDeviceToHost, sB));
    }
    BGP_CUDA(cudaEventRecord(h->ev[2], sB));  // ACA done
    BGP_CUDA(cudaStreamSynchronize(sB));

    // ---- ranks; grow the capacity of overflowing levels and repeat ----
    bool overflow = false;
    for (int i = 0; i < nint; ++i) {
      HNode& nd = h->nodes[desc_node[i]];
      nd.rank = houts[i].rank; nd.draws = houts[i].draws; nd.fallback = houts[i].fallback;
      if (houts[i].status == 2) { set_error("internal: ACA work list overflow"); return BGP_ERR_CUDA; }
      if (houts[i].status != 0) {
        LevelInfo& L = h->levels[nd.depth];
        if (o.rank_capacity > 0 || L.cap >= L.max_cap) {
          set_error("ACA rank capacity exceeded at node [start=%d size=%d] (capacity %d%s); raise rank_capacity", nd.start,
                    nd.size, L.cap, houts[i].fallback ? ", dense fallback" : "");
          return BGP_ERR_RANK_CAPACITY;
        }
        L.grow = houts[i].fallback ? L.max_cap : std::max(L.grow, std::min(L.max_cap, 2 * L.cap));
        overflow = true;
      }
    }
    if (!overflow) {
      h->cap_hint.assign(nlev, 0);
      for (int l = 0; l < nlev; ++l) h->cap_hint[l] = h->levels[l].cap;
      h->cap_hint_n = n; h->cap_hint_min_size = o.min_size;
      break;
    }
    for (auto& L : h->levels) if (L.grow > L.cap) L.cap = L.grow;
    if (attempt > 16) { set_error("ACA capacity growth did not converge"); return BGP_ERR_RANK_CAPACITY; }
  }
  int rtot_set[2] = {0, 0}, ndesc = 0, ndesc_top = 0;
  int64_t s_total = 0;
  size_t w_need = 1;
  std::vector<NodeDesc> hnd;
  for (int l = 0; l < nlev; ++l) {
    LevelInfo& L = h->levels[l];
    L.r = 0;
    for (int id : L.nodes) L.r = std::max(L.r, h->nodes[id].rank);
    L.ucol = rtot_set[L.set];
    rtot_set[L.set] += L.r;
    L.desc_off = ndesc;
    for (int id : L.nodes) {
      const HNode& nd = h->nodes[id];
      NodeDesc d;
      d.start = nd.start; d.size = nd.size; d.half = nd.half; d.depth = nd.depth; d.vcol = L.vcol; d.ucol = L.ucol;
      d.r = L.r; d.rank = nd.rank; d.s_off = s_total;
      s_total += (int64_t)(2 * L.r) * (2 * L.r) + 2 * L.r + 2;
      hnd.push_back(d);
      ndesc++;
      if (L.set == 0) ndesc_top++;
    }
    w_need = std::max(w_need, (size_t)L.nodes.size() * 2 * (size_t)L.r * (size_t)(L.ucol + L.r));
  }
  h->top.ucols = rtot_set[0]; h->loc.ucols = rtot_set[1];
  const int rtot = rtot_set[0] + rtot_set[1];
  h->rtot = rtot;
  // per-depth number of LOCAL ancestor columns a leaf (or node) at that depth sees (levels above the cut live in the top
  // panel set and receive this shard's sub-tree inverse in a separate pass, below)
  std::vector<int> ncols_by_depth(max_depth + 2, h->loc.ucols);
  for (int dpt = 0; dpt <= max_depth + 1; ++dpt)
    ncols_by_depth[dpt] = dpt < nlev ? (h->levels[dpt].set == 1 ? h->levels[dpt].ucol : 0) : h->loc.ucols;

  BGP_CUDA(cudaEventRecord(h->ev[6], sA));  // ranks known, both streams drained up to here: the up-sweep starts
  BGP_TRY(h->d_nodes.reserve(std::max(ndesc, 1), sA));
  BGP_TRY(h->d_node_logdet.reserve(std::max(ndesc, 1), sA));
  BGP_TRY(h->top.U.reserve((size_t)n * std::max(h->top.ucols, 1), sA));
  BGP_TRY(h->loc.U.reserve((size_t)h->nloc * std::max(h->loc.ucols, 1), sA));
  BGP_TRY(h->d_S.reserve((size_t)std::max<int64_t>(s_total, 1), sA));
  // solve() needs 2*r*nrhs per node; keep room for 64 right-hand sides per batch
  for (auto& L : h->levels) w_need = std::max(w_need, (size_t)L.nodes.size() * 2 * (size_t)L.r * 64);
  BGP_TRY(h->d_W.reserve(w_need, sA));
  h->w_cap = h->d_W.n;
  BGP_TRY(h->d_ncols_by_depth.reserve(ncols_by_depth.size(), sA));
  BGP_TRY(h->d_scalar.reserve(4, sA));
  BGP_CUDA(cudaMemcpyAsync(h->d_ncols_by_depth.p, ncols_by_depth.data(), sizeof(int) * ncols_by_depth.size(), cudaMemcpyHostToDevice, sA));
  if (ndesc) {
    BGP_CUDA(cudaMemcpyAsync(h->d_nodes.p, hnd.data(), sizeof(NodeDesc) * ndesc, cudaMemcpyHostToDevice, sA));
    h->h_nodes = hnd;
    BGP_CUDA(cudaMemsetAsync(h->d_node_logdet.p, 0, sizeof(double) * ndesc, sA));
    // the levels above the cut come first in the descriptor list: one launch per panel set, over FP_ROWS-row tiles of
    // the nodes of rank > 0
    std::vector<PanelTile> tiles;
    int ntiles_top = 0;
    for (int i = 0; i < ndesc; ++i) {
      if (i == ndesc_top) ntiles_top = (int)tiles.size();
      if (hnd[i].r == 0) continue;
      for (int r0 = 0; r0 < hnd[i].size; r0 += FP_ROWS) tiles.push_back(PanelTile{i, r0});
    }
    if (ndesc_top == ndesc) ntiles_top = (int)tiles.size();
    const int ntiles = (int)tiles.size();
    if (ntiles > 0) {
      BGP_TRY(h->d_ptiles.reserve(ntiles, sA));
      BGP_CUDA(cudaMemcpyAsync(h->d_ptiles.p, tiles.data(), sizeof(PanelTile) * ntiles, cudaMemcpyHostToDevice, sA));
    }
    if (ntiles_top > 0) {
      finalize_panels_kernel<<<ntiles_top, FP_THREADS, 0, sA>>>(h->d_nodes.p, h->d_ptiles.p, h->top.vbase(), h->top.ld,
                                                                h->top.ubase(), h->top.ld);
      BGP_LAUNCH_CHECK();
    }
    if (ntiles > ntiles_top) {
      finalize_panels_kernel<<<ntiles - ntiles_top, FP_THREADS, 0, sA>>>(h->d_nodes.p, h->d_ptiles.p + ntiles_top,
                                                                         h->loc.vbase(), h->loc.ld, h->loc.ubase(), h->loc.ld);
      BGP_LAUNCH_CHECK();
    }
  }

  // ---- up-sweep (stream A; leaves are already ordered before this on the same stream) ----
  // (1) the owned sub-tree against its own (local) ancestor columns
  if (h->loc.ucols > 0) BGP_TRY(launch_leaf_solve(h, h->loc.ubase(), h->loc.ld, h->d_ncols_by_depth.p, 0, h->loc.ucols, sA));
  const int stop_level = (o.shard_count > 1) ? h->cut_depth : 0;
  for (int l = nlev - 1; l >= stop_level; --l) {
    const LevelInfo& L = h->levels[l];
    BGP_TRY(launch_level(h, L, h->loc.ubase(), h->loc.ld, L.ucol + L.r, L.ucol, 1, 0, L.ucol, sA));
  }
  // (2) sharded: the factored sub-tree applied to this shard's rows of the top-level factor columns (hodlr.h:95-102 for
  //     the ancestors above the cut) — the same kernels as a solve with the top panel as right-hand sides
  if (o.shard_count > 1 && h->top.ucols > 0) BGP_TRY(hodlr_solve_dev(h, h->top.U.p, h->top.ucols, n, sA, 1));
  BGP_CUDA(cudaEventRecord(h->ev[3], sA));
  if (o.shard_count > 1) {
    if (!host_exchange(h)) return hodlr_exchange_finish(h);
    // no communicator: the caller exchanges the top panel rows itself and calls bgp_hodlr_finish_top()
    BGP_CUDA(cudaStreamSynchronize(sA));
    h->top_pending = true;
    return BGP_OK;
  }

  // ---- log-det ----
  std::vector<double> ld_leaf(nl), ld_node(ndesc);
  if (nl) BGP_CUDA(cudaMemcpyAsync(ld_leaf.data(), h->d_leaf_logdet.p, sizeof(double) * nl, cudaMemcpyDeviceToHost, sA));
  if (ndesc) BGP_CUDA(cudaMemcpyAsync(ld_node.data(), h->d_node_logdet.p, sizeof(double) * ndesc, cudaMemcpyDeviceToHost, sA));
  if (nint) {
    h->h_piv_rows.resize(piv_total); h->h_piv_cols.resize(piv_total);
  }
  BGP_CUDA(cudaStreamSynchronize(sA));
  double ld = 0.0;
  for (double v : ld_leaf) ld += v;
  for (double v : ld_node) ld += v;
  h->log_det = ld;
  h->computed = true;

  float ms = 0;
  cudaEventElapsedTime(&ms, h->ev[0], h->ev[1]); h->t_ms[0] = ms;
  cudaEventElapsedTime(&ms, h->ev[0], h->ev[2]); h->t_ms[1] = ms;
  cudaEventElapsedTime(&ms, h->ev[6], h->ev[3]); h->t_ms[2] = ms;  // panel finalisation + leaf solves + level sweeps only
  cudaEventElapsedTime(&ms, h->ev[0], h->ev[3]); h->t_ms[3] = ms;

  // algorithmic work (SURVEY.md §8d)
  {
    double evals = 0, bytes = 0, flops = 0, R = rtot;
    for (int id : h->leaves) { const double m = h->nodes[id].size; evals += m * (m + 1) / 2; bytes += 8 * m * m; flops += m * m * m / 3 + 2 * m * m * ncols_by_depth[h->nodes[id].depth]; }
    for (int l = 0; l < nlev; ++l) {
      const LevelInfo& L = h->levels[l];
      for (int id : L.nodes) {
        const HNode& nd = h->nodes[id];
        evals += (double)nd.size * nd.draws;  // one row + one column of the block per accepted/rejected draw (upper bound)
        bytes += 16.0 * nd.size * nd.rank;
        flops += 4.0 * nd.size * L.r * L.ucol + 2.0 * nd.size * L.r * L.r + 2.0 * nd.size * nd.rank * nd.rank;
      }
    }
    h->work[0] = evals; h->work[1] = bytes; h->work[2] = flops; h->work[3] = R; h->work[4] = h->max_leaf; h->work[5] = nlev;
  }
  return BGP_OK;
}

// all-gather of the shards' row slices of `cols` columns of a column-major matrix P (leading dimension ld): every rank
// ends up with all rows.  pack -> ncclAllGather -> unpack on one stream, no host synchronisation.
static int exchange_rows(bgp_hodlr* h, double* P, int64_t ld, int64_t cols, cudaStream_t s) {
  if (cols <= 0) return BGP_OK;
  const int world = h->opts.shard_count;
  int64_t rows_pad = 0;
  for (int64_t r : h->shard_rows) rows_pad = std::max(rows_pad, r);
  const size_t per = (size_t)cols * rows_pad;
  BGP_TRY(h->d_xsend.reserve(per, s));
  BGP_TRY(h->d_xrecv.reserve(per * world, s));
  if (h->nloc < rows_pad) BGP_CUDA(cudaMemsetAsync(h->d_xsend.p, 0, sizeof(double) * per, s));
  pack_rows_kernel<<<1184, 256, 0, s>>>(P, ld, h->row0, h->nloc, cols, h->d_xsend.p, rows_pad);
  BGP_LAUNCH_CHECK();
  BGP_TRY(comm_allgather_f64(h->d_xsend.p, h->d_xrecv.p, per, s));
  for (int sh = 0; sh < world; ++sh) {
    if (sh == h->opts.shard_rank) continue;  // own rows are already in place
    unpack_rows_kernel<<<1184, 256, 0, s>>>(P, ld, h->shard_row0[sh], h->shard_rows[sh], cols, h->d_xrecv.p + (size_t)sh * per, rows_pad);
    BGP_LAUNCH_CHECK();
  }
  return BGP_OK;
}

// exchange_rows for an n x cols ROW-major matrix P (dx of bgp_hodlr_grad_x_terms): through a column-major copy
__global__ void transpose_rows_kernel(const double* __restrict__ src, int64_t rows, int64_t cols, double* __restrict__ dst) {
  const int64_t total = rows * cols;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / cols, q = t - i * cols;
    dst[q * rows + i] = src[t];
  }
}
static int exchange_rows_wide(bgp_hodlr* h, double* P, int64_t cols, cudaStream_t s) {
  if (cols == 1) return exchange_rows(h, P, h->n, 1, s);
  const int64_t n = h->n, total = n * cols;
  const unsigned blocks = (unsigned)std::min<int64_t>((total + 255) / 256, 1184);
  DevBuf<double> colmajor;
  BGP_TRY(colmajor.alloc((size_t)total, s));
  transpose_rows_kernel<<<blocks, 256, 0, s>>>(P, n, cols, colmajor.p);
  BGP_LAUNCH_CHECK();
  BGP_TRY(exchange_rows(h, colmajor.p, n, cols, s));
  transpose_rows_kernel<<<blocks, 256, 0, s>>>(colmajor.p, cols, n, P);  // column-major n x cols = row-major cols x n
  BGP_LAUNCH_CHECK();
  return BGP_OK;
}

// [*first, *last): the items 0 .. count-1, whose row intervals [start(k), start(k) + size(k)) are disjoint and ordered
// by start, that meet rows [lo, hi)
template <class StartSize>
static void rows_meeting(int count, const StartSize& start_size, int64_t lo, int64_t hi, int* first, int* last) {
  int a = 0, b = count;  // first item ending after lo
  while (a < b) {
    const int m = (a + b) / 2;
    int st, sz;
    start_size(m, &st, &sz);
    if ((int64_t)st + sz <= lo) a = m + 1; else b = m;
  }
  *first = a;
  b = count;  // first item starting at or after hi
  while (a < b) {
    const int m = (a + b) / 2;
    int st, sz;
    start_size(m, &st, &sz);
    if (st < hi) a = m + 1; else b = m;
  }
  *last = a;
}

// Leaves (h->leaves) and each level's nodes (L.nodes, and so its NodeDesc block) are in pre-order, which lists the
// disjoint row intervals of one depth, and the leaves, from left to right: rows_meeting's precondition.
static bool rows_ordered(const bgp_hodlr* h) {
  auto ordered = [&](const std::vector<int>& ids) {
    for (size_t k = 1; k < ids.size(); ++k) {
      const HNode& a = h->nodes[ids[k - 1]];
      if (a.start + a.size > h->nodes[ids[k]].start) return false;
    }
    return true;
  };
  if (!ordered(h->leaves)) return false;
  for (const LevelInfo& L : h->levels)
    if (!ordered(L.nodes)) return false;
  return true;
}

// part: 0 = everything, 1 = local (leaves + levels >= cut), 2 = top (levels < cut)
// eye_row0 >= 0 restricts the solve by rows: the caller guarantees that columns [c0, c0 + 64) of b are zero outside rows
// [eye_row0 + c0, eye_row0 + c0 + 64) (identity columns e_j, j = eye_row0 + column: grad_terms' K^-1 slabs).  Every step
// of the solve is block diagonal and maps zero rows to zero rows, so only the leaves and, per level, the nodes that meet
// those rows run; the result is bit for bit the unrestricted one.  Part 0 only.
// On a shard the caller also guarantees that b is zero outside the shard's rows [row0, row0 + nloc), so the identity
// rows are clamped to them: the other shards' sub-tree solves of such columns are zero.  The owned leaves and levels then
// run through the local panel set, the levels above the cut through the top panels (all N rows, identical on every shard
// after finish_top), and no rows are exchanged: a restricted solve issues no collective, so shards that run different
// numbers of slabs cannot block each other.
static int hodlr_solve_dev(bgp_hodlr* h, double* b, int64_t nrhs, int64_t ldb, cudaStream_t s, int part,
                           int64_t eye_row0) {
  const int nlev = (int)h->levels.size();
  const int cut = h->opts.shard_count > 1 ? h->cut_depth : 0;
  const bool native_x = part == 0 && h->opts.shard_count > 1 && !host_exchange(h);
  if (eye_row0 >= 0 && part != 0) {
    set_error("internal: a row-restricted solve runs every part of the solve");
    return BGP_ERR_INVALID;
  }
  for (int64_t c0 = 0; c0 < nrhs; c0 += 64) {
    const int nc = (int)std::min<int64_t>(64, nrhs - c0);
    double* X = b + c0 * ldb;
    if (eye_row0 >= 0) {
      const int64_t lo = std::max(eye_row0 + c0, h->row0), hi = std::min(eye_row0 + c0 + nc, h->row0 + h->nloc);
      if (lo >= hi) continue;  // no identity row of this handle's: the group stays zero
      int l0, l1;
      rows_meeting((int)h->leaves.size(), [&](int k, int* st, int* sz) {
        const HNode& nd = h->nodes[h->leaves[k]]; *st = nd.start; *sz = nd.size; }, lo, hi, &l0, &l1);
      BGP_TRY(launch_leaf_solve(h, X, ldb, nullptr, nc, nc, s, l0, l1));
      for (int l = nlev - 1; l >= 0; --l) {
        const LevelInfo& L = h->levels[l];
        int b0, b1;
        rows_meeting((int)L.nodes.size(), [&](int k, int* st, int* sz) {
          const HNode& nd = h->nodes[L.nodes[k]]; *st = nd.start; *sz = nd.size; }, lo, hi, &b0, &b1);
        BGP_TRY(launch_level(h, L, X, ldb, nc, 0, 0, 0, nc, s, b0, b1));
      }
      continue;
    }
    if (part != 2) {
      BGP_TRY(launch_leaf_solve(h, X, ldb, nullptr, nc, nc, s));
      for (int l = nlev - 1; l >= cut; --l) BGP_TRY(launch_level(h, h->levels[l], X, ldb, nc, 0, 0, 0, nc, s));
    }
    if (native_x) BGP_TRY(exchange_rows(h, X, ldb, nc, s));  // replicated right-hand side: every rank needs all rows
    if (part != 1) {
      for (int l = std::min(cut, nlev) - 1; l >= 0; --l) BGP_TRY(launch_level(h, h->levels[l], X, ldb, nc, 0, 0, 0, nc, s));
    }
  }
  return BGP_OK;
}

static int64_t top_cols(const bgp_hodlr_t* h) {
  const int cut = std::min<int>(h->cut_depth, (int)h->levels.size());
  (void)cut;
  return h->top.ucols;
}

// Gram / LU / log-det / update of the nodes above the shard cut (every rank does all of them: they are tiny), then the
// log-determinant: owned leaves + owned nodes, the top nodes counted once (by shard 0); with `allreduce` the partial sums
// are added over the ranks on the device (one double), otherwise log_det stays PARTIAL and the host sums over shards.
static int hodlr_finish_top_impl(bgp_hodlr* h, bool allreduce) {
  cudaStream_t s = h->sA;
  const int nlev = (int)h->levels.size();
  const int cut = std::min(h->cut_depth, nlev);
  for (int l = cut - 1; l >= 0; --l) {
    const LevelInfo& L = h->levels[l];
    BGP_TRY(launch_level(h, L, h->top.U.p, h->n, L.ucol + L.r, L.ucol, 1, 0, L.ucol, s));
  }
  const int nl = (int)h->leaves.size();
  int ndesc = 0;
  for (auto& L : h->levels) ndesc += (int)L.nodes.size();
  std::vector<double> ld_leaf(nl), ld_node(ndesc);
  if (nl) BGP_CUDA(cudaMemcpyAsync(ld_leaf.data(), h->d_leaf_logdet.p, sizeof(double) * nl, cudaMemcpyDeviceToHost, s));
  if (ndesc) BGP_CUDA(cudaMemcpyAsync(ld_node.data(), h->d_node_logdet.p, sizeof(double) * ndesc, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  double ld = 0.0;
  for (double v : ld_leaf) ld += v;
  for (int l = 0; l < nlev; ++l) {
    const LevelInfo& L = h->levels[l];
    if (l < cut && h->opts.shard_rank != 0) continue;
    for (size_t i = 0; i < L.nodes.size(); ++i) ld += ld_node[L.desc_off + i];
  }
  if (allreduce) {
    BGP_CUDA(cudaMemcpyAsync(h->d_scalar.p, &ld, sizeof(double), cudaMemcpyHostToDevice, s));
    BGP_TRY(comm_allreduce_sum_f64(h->d_scalar.p, 1, s));
    BGP_CUDA(cudaMemcpyAsync(&ld, h->d_scalar.p, sizeof(double), cudaMemcpyDeviceToHost, s));
    BGP_CUDA(cudaStreamSynchronize(s));
  }
  h->log_det = ld;
  h->computed = true;
  return BGP_OK;
}

// sharded compute with the library's communicator: all-gather of the locally solved rows of the top-level factor panel
// (the ONE data-path collective of compute(), SURVEY.md §8e), then the top nodes, then the log-det all-reduce.
static int hodlr_exchange_finish(bgp_hodlr* h) {
  BGP_TRY(exchange_rows(h, h->top.U.p, h->n, top_cols(h), h->sA));
  BGP_TRY(hodlr_finish_top_impl(h, true));
  float ms = 0;
  cudaEventElapsedTime(&ms, h->ev[0], h->ev[1]); h->t_ms[0] = ms;
  cudaEventElapsedTime(&ms, h->ev[0], h->ev[2]); h->t_ms[1] = ms;
  cudaEventElapsedTime(&ms, h->ev[6], h->ev[3]); h->t_ms[2] = ms;
  cudaEventElapsedTime(&ms, h->ev[0], h->ev[3]); h->t_ms[3] = ms;
  return BGP_OK;
}

extern "C" {

void bgp_hodlr_default_opts(bgp_hodlr_opts_t* o) {
  o->min_size = 100; o->seed = 42; o->tol = 0.1;  // _hodlr.cpp:202
  o->rng_mode = BGP_RNG_REFERENCE;  // at the default tol the answer depends on the pivots: reproduce the reference's order
  o->rank_capacity = 0; o->shard_rank = 0; o->shard_count = 1; o->exhaust_mode = BGP_EXHAUST_DENSE;
}

int bgp_hodlr_create(bgp_hodlr_t** out) {
  *out = new (std::nothrow) bgp_hodlr();
  if (!*out) { set_error("out of host memory"); return BGP_ERR_NOMEM; }
  bgp_hodlr_default_opts(&(*out)->opts);
  return BGP_OK;
}

void bgp_hodlr_destroy(bgp_hodlr_t* h) {
  if (!h) return;
  if (h->sA) {
    cudaStreamSynchronize(h->sA); cudaStreamSynchronize(h->sB);
  }
  // release buffers while the streams are still alive
  h->d_prog.release(); h->d_x.release(); h->d_yerr.release(); h->d_diag.release(); h->d_L.release();
  h->d_leaf_logdet.release(); h->d_node_logdet.release(); h->top.V.release(); h->top.U.release(); h->loc.V.release(); h->loc.U.release(); h->d_S.release();
  h->d_W.release(); h->d_scalar.release(); h->d_rhs.release(); h->d_leaves.release(); h->d_aca.release();
  h->d_aca_out.release(); h->d_nodes.release(); h->d_ptiles.release(); h->d_idx.release(); h->d_piv_rows.release(); h->d_piv_cols.release();
  h->lu_ws.d_nodes.release(); h->lu_ws.d_trsm.release(); h->lu_ws.d_gemm.release(); h->d_gram_desc.release(); h->d_upd_desc.release();
  h->d_ticket.release(); h->d_chain_done.release(); h->d_ncols_by_depth.release(); h->d_chain_state.release();
  h->d_a2nodes.release(); h->d_a2states.release(); h->d_a2rngs.release(); h->d_epart.release(); h->d_cand.release(); h->d_cand_k.release();
  h->d_cand_words.release(); h->d_cand_L.release(); h->d_cand_next.release(); h->d_cand_live.release(); h->d_node_box.release(); h->d_cand_xu.release(); h->d_gbox.release(); h->d_cbox.release(); h->d_cchunk_node.release(); h->d_rchunk_node.release(); h->d_nactive.release();
  h->d_inv.release(); h->d_gscratch.release(); h->d_which.release(); h->d_xsend.release(); h->d_xrecv.release();
  h->d_vpart.release(); h->d_upart.release(); h->d_vmax.release(); h->d_cmax.release(); h->d_stats.release(); h->d_work.release(); h->d_work_count.release();
  for (cudaEvent_t e : h->prof_events) cudaEventDestroy(e);
  h->d_iter.release();
  if (h->sym) sym_destroy(h->sym);
  if (h->aca_exec) cudaGraphExecDestroy(h->aca_exec);
  if (h->aca_graph) cudaGraphDestroy(h->aca_graph);
  if (h->sC) cudaStreamDestroy(h->sC);
  if (h->sA) {
    cudaStreamSynchronize(h->sA); cudaStreamSynchronize(h->sB);
    for (int i = 0; i < 8; ++i) cudaEventDestroy(h->ev[i]);
    cudaStreamDestroy(h->sA); cudaStreamDestroy(h->sB);
  }
  delete h;
}

int bgp_hodlr_compute_dev(bgp_hodlr_t* h, const bgp_kernel_spec_t* spec, const double* x_dev, int64_t n, int32_t ndim,
                          const double* yerr_dev, const bgp_hodlr_opts_t* opts) {
  if (!h) { set_error("null handle"); return BGP_ERR_INVALID; }
  return hodlr_compute_dev_impl(h, spec, x_dev, n, ndim, yerr_dev, opts);
}

int bgp_hodlr_compute(bgp_hodlr_t* h, const bgp_kernel_spec_t* spec, const double* x, int64_t n, int32_t ndim,
                      const double* yerr, const bgp_hodlr_opts_t* opts) {
  if (!h) { set_error("null handle"); return BGP_ERR_INVALID; }
  h->computed = false;
  h->sym_current = false;
  h->sym_stage = 0;
  h->top_pending = false;  // (hodlr_compute_dev_impl resets these too; this covers the returns before it)
  h->shard_row0.clear(); h->shard_rows.clear();
  BGP_TRY(require_device());
  BGP_TRY(ensure_streams(h));
  if (n <= 0 || ndim <= 0) { set_error("invalid input shape (%lld, %d)", (long long)n, ndim); return BGP_ERR_INVALID; }
  BGP_TRY(h->d_x.reserve((size_t)n * ndim, h->sA));
  BGP_TRY(h->d_yerr.reserve((size_t)n, h->sA));
  BGP_CUDA(cudaMemcpyAsync(h->d_x.p, x, sizeof(double) * n * ndim, cudaMemcpyHostToDevice, h->sA));
  BGP_CUDA(cudaMemcpyAsync(h->d_yerr.p, yerr, sizeof(double) * n, cudaMemcpyHostToDevice, h->sA));
  return hodlr_compute_dev_impl(h, spec, h->d_x.p, n, ndim, h->d_yerr.p, opts);
}

int bgp_hodlr_computed(const bgp_hodlr_t* h) { return h && h->computed ? 1 : 0; }

int bgp_hodlr_log_determinant(const bgp_hodlr_t* h, double* out) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  *out = h->log_det;
  return BGP_OK;
}

int bgp_hodlr_apply_inverse(bgp_hodlr_t* h, double* b, int64_t nrhs, int64_t ldb) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  BGP_TRY(reject_host_exchange(h, "apply_inverse"));
  if (nrhs <= 0) return BGP_OK;
  if (ldb < h->n) { set_error("dimension mismatch: ldb < n"); return BGP_ERR_DIM; }
  cudaStream_t s = h->sA;
  const int64_t n = h->n;
  // process in slabs of columns to bound device memory
  const int64_t slab = std::max<int64_t>(1, std::min<int64_t>(nrhs, (int64_t)(1ull << 28) / n));
  BGP_TRY(h->d_rhs.reserve((size_t)n * slab, s));
  for (int64_t c0 = 0; c0 < nrhs; c0 += slab) {
    const int64_t nc = std::min(slab, nrhs - c0);
    BGP_CUDA(cudaMemcpy2DAsync(h->d_rhs.p, sizeof(double) * n, b + c0 * ldb, sizeof(double) * ldb, sizeof(double) * n, nc, cudaMemcpyHostToDevice, s));
    BGP_CUDA(cudaEventRecord(h->ev[4], s));
    BGP_TRY(hodlr_solve_dev(h, h->d_rhs.p, nc, n, s, 0));
    BGP_CUDA(cudaEventRecord(h->ev[5], s));
    BGP_CUDA(cudaMemcpy2DAsync(b + c0 * ldb, sizeof(double) * ldb, h->d_rhs.p, sizeof(double) * n, sizeof(double) * n, nc, cudaMemcpyDeviceToHost, s));
    BGP_CUDA(cudaStreamSynchronize(s));
  }
  float ms = 0; cudaEventElapsedTime(&ms, h->ev[4], h->ev[5]); h->t_ms[4] = ms;
  return BGP_OK;
}

int bgp_hodlr_dot_solve_dev(bgp_hodlr_t* h, const double* y_dev, double* out) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  BGP_TRY(reject_host_exchange(h, "dot_solve"));
  cudaStream_t s = h->sA;
  const int64_t n = h->n;
  BGP_TRY(h->d_rhs.reserve((size_t)n, s));
  BGP_CUDA(cudaEventRecord(h->ev[4], s));
  BGP_CUDA(cudaMemcpyAsync(h->d_rhs.p, y_dev, sizeof(double) * n, cudaMemcpyDeviceToDevice, s));
  BGP_TRY(hodlr_solve_dev(h, h->d_rhs.p, 1, n, s, 0));
  BGP_CUDA(cudaMemsetAsync(h->d_scalar.p, 0, sizeof(double), s));
  dot_kernel<<<(unsigned)std::min<int64_t>((n + 255) / 256, 592), 256, 0, s>>>(y_dev, h->d_rhs.p, n, h->d_scalar.p);
  BGP_LAUNCH_CHECK();
  BGP_CUDA(cudaEventRecord(h->ev[5], s));
  BGP_CUDA(cudaMemcpyAsync(out, h->d_scalar.p, sizeof(double), cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  float ms = 0; cudaEventElapsedTime(&ms, h->ev[4], h->ev[5]); h->t_ms[4] = ms;
  return BGP_OK;
}

int bgp_hodlr_dot_solve(bgp_hodlr_t* h, const double* y, double* out) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  BGP_TRY(reject_host_exchange(h, "dot_solve"));
  cudaStream_t s = h->sA;
  BGP_TRY(h->d_yerr.reserve((size_t)h->n, s));  // reuse as staging for y
  BGP_CUDA(cudaMemcpyAsync(h->d_yerr.p, y, sizeof(double) * h->n, cudaMemcpyHostToDevice, s));
  return bgp_hodlr_dot_solve_dev(h, h->d_yerr.p, out);
}

int bgp_hodlr_get_inverse(bgp_hodlr_t* h, double* out) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  BGP_TRY(reject_host_exchange(h, "get_inverse"));
  const int64_t n = h->n;
  for (int64_t j = 0; j < n; ++j) {
    double* c = out + j * n;
    memset(c, 0, sizeof(double) * n);
    c[j] = 1.0;
  }
  return bgp_hodlr_apply_inverse(h, out, n, n);  // COLUMN-major K^-1 (symmetric only to tol: the host transposes)
}

// E_J: columns j0 .. j0 + nc of the identity, n rows, where j0 + k lies in [jlo, jhi); the other columns stay zero (the
// slab W is zeroed before)
__global__ void eye_slab_kernel(double* __restrict__ W, int64_t n, int64_t j0, int64_t nc, int64_t jlo, int64_t jhi) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nc; k += (int64_t)gridDim.x * blockDim.x)
    if (j0 + k >= jlo && j0 + k < jhi) W[k * n + j0 + k] = 1.0;
}

// K^-1 resident (n x n) up to this many doubles (n <= 65536); larger n streams it in column slabs
constexpr int64_t GRAD_RESIDENT_MAX = (int64_t)1 << 32;
constexpr int64_t GRAD_SLAB_BUDGET = (int64_t)1 << 27;  // doubles (1 GiB) per K^-1 slab

// Columns per K^-1 slab: as many n-row columns as fit in GRAD_SLAB_BUDGET, at least 64, a multiple of 64 (the
// predict_chunk_cols rule).  BGP_GRAD_CHUNK=<c> (read at every call, like BGP_PREDICT_CHUNK) forces the streamed path at
// any n with c columns, rounded up to 64; tests use it to run many slabs with a ragged tail at small sizes.
static int64_t grad_slab_cols(int64_t n, bool* forced) {
  int64_t c = std::max<int64_t>(64, (GRAD_SLAB_BUDGET / std::max<int64_t>(n, 1)) / 64 * 64);
  *forced = false;
  if (const char* e = getenv("BGP_GRAD_CHUNK")) {
    const long v = atol(e);
    if (v >= 1) { c = (v + 63) / 64 * 64; *forced = true; }
  }
  return std::min(c, (n + 63) / 64 * 64);
}

static float event_ms(cudaEvent_t a, cudaEvent_t b) {
  float ms = 0;
  cudaEventElapsedTime(&ms, a, b);
  return ms;
}

// The streamed gradient over this handle's own columns J = [row0, row0 + nloc) ([0, n) unsharded, a shard's rows):
//     dg_p = sum_{i, j in J} (alpha_i alpha_j - K^-1_ij) dK_ij/dtheta_p,   ddiag_j = alpha_j^2 - K^-1_jj (j in J only).
// Slabs of c columns start at the global multiple of 64 at or below row0; the identity is placed in J only, each slab is
// solved with the row-restricted solve and contracted over the window J, and the per-tile partials of the tiles meeting
// J are summed in order.  alpha: the full n-vector K^-1 r; d_which holds which[0 .. np).  Issues no collective.
// ddx (may be NULL): each slab also contracts the input gradient of its columns in the same pass
// (kmat_grad_x_slab_launch), ddx[j * ndim + q] for j in J only; g and ddiag keep their bits.
static int grad_stream_own_columns(bgp_hodlr* h, int np, const double* alpha, int64_t c, double* dg, double* ddiag,
                                   double* t_solve, double* t_contract, double* ddx = nullptr) {
  cudaStream_t s = h->sA;
  const int64_t n = h->n, jlo = h->row0, jhi = h->row0 + h->nloc;
  const bool prof = h->profile;
  // slab W (n x c), then the per-tile partials, one slab's per-split partials and (ddx) its input-gradient partials in
  // d_gscratch
  const int64_t tsize = grad_slab_tile_size(n, np), psize = grad_slab_partial_size(n, c, np);
  const int64_t xsize = ddx ? grad_slab_x_partial_size(n, c, h->ndim) : 0;
  BGP_TRY(h->d_inv.reserve((size_t)n * c, s));
  BGP_TRY(h->d_gscratch.reserve((size_t)(tsize + psize + xsize), s));
  double* W = h->d_inv.p;
  double* tile_part = h->d_gscratch.p;
  double* partial = h->d_gscratch.p + tsize;
  double* xpart = partial + psize;
  int64_t slabs = 0;
  for (int64_t j0 = jlo / 64 * 64; j0 < jhi; j0 += c, ++slabs) {
    const int64_t nc = std::min(c, jhi - j0);
    if (prof) BGP_CUDA(cudaEventRecord(h->ev[4], s));
    BGP_CUDA(cudaMemsetAsync(W, 0, sizeof(double) * n * nc, s));
    eye_slab_kernel<<<(unsigned)std::min<int64_t>((nc + 255) / 256, 1184), 256, 0, s>>>(W, n, j0, nc, jlo, jhi);
    BGP_LAUNCH_CHECK();
    BGP_TRY(hodlr_solve_dev(h, W, nc, n, s, 0, j0));
    if (prof) BGP_CUDA(cudaEventRecord(h->ev[5], s));
    if (ddx)
      BGP_TRY(kmat_grad_x_slab_launch(h->d_prog.p, h->prog.shape, h->ndim, np, h->d_which.p, h->d_x.p, n, W, j0, nc, jlo,
                                      jhi, alpha, partial, tile_part, xpart, ddiag, ddx, s));
    else
      BGP_TRY(kmat_grad_slab_launch(h->d_prog.p, h->ndim, np, h->d_which.p, h->d_x.p, n, W, j0, nc, jlo, jhi, alpha,
                                    alpha, partial, tile_part, ddiag, s));
    if (prof) {
      BGP_CUDA(cudaEventRecord(h->ev[7], s));
      BGP_CUDA(cudaEventSynchronize(h->ev[7]));
      *t_solve += event_ms(h->ev[4], h->ev[5]);
      *t_contract += event_ms(h->ev[5], h->ev[7]);
    }
  }
  if (prof) BGP_CUDA(cudaEventRecord(h->ev[4], s));
  BGP_TRY(kmat_grad_slab_finish(np, jlo, jhi, tile_part, dg, s));
  if (prof) {
    BGP_CUDA(cudaEventRecord(h->ev[5], s));
    BGP_CUDA(cudaEventSynchronize(h->ev[5]));
    *t_contract += event_ms(h->ev[4], h->ev[5]);
  }
  h->grad_t[2] = (double)slabs;
  h->grad_t[3] = (double)c;
  return BGP_OK;
}

// alpha = K^-1 r, g_p = sum_ij (alpha alpha^T - K^-1)_ij dK_ij/dtheta_p, diag(alpha alpha^T - K^-1): everything
// GP.grad_log_likelihood (gp.py:406-468) needs from the solver, with K^-1 (solve against the identity, _hodlr.cpp:193-199)
// and the gradient contraction staying on the device.
// Two regimes (include/bgp.h): up to n = 65536 K^-1 is formed whole and contracted by kmat_grad_contract_kernel; above,
// or with BGP_GRAD_CHUNK set, it is streamed in column slabs W = K^-1 E_J, each solved with the row-restricted solve
// and contracted by kmat_grad_slab_kernel, so K^-1 is never resident.
// On a shard with a matching communicator the call is collective and always streamed, composed of the existing pieces:
// alpha by the collective solve, grad_stream_own_columns on this shard's columns, an all-reduce of g and an all-gather
// of the diag slices.  Every rank issues the same collectives in the same order; none sits inside the slab loop.
// With xgrad (bgp_hodlr_grad_x_terms) the same call also forms dx (n x ndim, row-major): resident, by the x-gradient
// matvec over alpha alpha^T - K^-1 after the contraction; streamed, in the slabs' own pass; sharded, one more all-gather
// of the dx row slices.  A NULL `which` then skips the parameter contraction.
static int hodlr_grad_terms_impl(bgp_hodlr* h, const uint32_t* which, const double* r, double* alpha_out, double* g_out,
                                 double* diag_out, bool xgrad, double* dx_out, const char* what) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  if (host_exchange(h)) { set_error("%s is not available on a sharded factorisation", what); return BGP_ERR_INVALID; }
  const int64_t n = h->n;
  const int np = (xgrad && !which) ? 0 : h->prog.n_params_total;
  if (np > 64) { set_error("gradient supports at most 64 hyper-parameters"); return BGP_ERR_INVALID; }
  const int nd = h->ndim;
  if (xgrad && nd > BGP_MAX_DIM) { set_error("input-coordinate gradients support at most %d dimensions (got %d)", BGP_MAX_DIM, nd); return BGP_ERR_INVALID; }
  const bool sharded = h->opts.shard_count > 1;
  if (sharded && !rows_ordered(h)) { set_error("internal: HODLR rows are not ordered by level"); return BGP_ERR_CUDA; }
  cudaStream_t s = h->sA;
  bool forced = false;
  const int64_t c = grad_slab_cols(n, &forced);
  const bool resident = !sharded && !forced && n * n <= GRAD_RESIDENT_MAX;
  const bool prof = h->profile;
  double t_solve = 0, t_contract = 0;
  for (double& t : h->grad_t) t = 0;
  BGP_TRY(h->d_rhs.reserve((size_t)n * 2 + 64, s));
  double* alpha = h->d_rhs.p;
  double* dg = h->d_rhs.p + n;
  double* ddiag = h->d_rhs.p + n + 64;
  BGP_CUDA(cudaMemcpyAsync(alpha, r, sizeof(double) * n, cudaMemcpyHostToDevice, s));
  if (prof) BGP_CUDA(cudaEventRecord(h->ev[4], s));
  BGP_TRY(hodlr_solve_dev(h, alpha, 1, n, s, 0));
  if (prof) { BGP_CUDA(cudaEventRecord(h->ev[5], s)); BGP_CUDA(cudaEventSynchronize(h->ev[5])); t_solve += event_ms(h->ev[4], h->ev[5]); }
  if (alpha_out) BGP_CUDA(cudaMemcpyAsync(alpha_out, alpha, sizeof(double) * n, cudaMemcpyDeviceToHost, s));
  DevBuf<double> ddx;
  if (xgrad) BGP_TRY(ddx.alloc((size_t)n * nd, s));
  if (resident) {
    if (prof) BGP_CUDA(cudaEventRecord(h->ev[4], s));
    BGP_TRY(h->d_inv.reserve((size_t)n * n, s));
    BGP_TRY(fill_identity_launch(h->d_inv.p, n, s));
    BGP_TRY(hodlr_solve_dev(h, h->d_inv.p, n, n, s, 0));
    if (prof) BGP_CUDA(cudaEventRecord(h->ev[5], s));
    BGP_TRY(h->d_which.reserve(std::max(np, 1), s));
    if (np) BGP_CUDA(cudaMemcpyAsync(h->d_which.p, which, sizeof(unsigned) * np, cudaMemcpyHostToDevice, s));
    BGP_TRY(kmat_grad_contract_launch(h->d_prog.p, h->ndim, np, h->d_which.p, h->d_x.p, n, h->d_inv.p, n, alpha, 1.0, -1.0, dg,
                                      diag_out ? ddiag : nullptr, h->d_gscratch, s));
    if (xgrad) BGP_TRY(grad_x_resident_launch(h->prog, h->d_prog.p, h->d_x.p, n, h->d_inv.p, alpha, ddx.p, h->d_gscratch, s));
    if (prof) {
      BGP_CUDA(cudaEventRecord(h->ev[7], s));
      BGP_CUDA(cudaEventSynchronize(h->ev[7]));
      t_solve += event_ms(h->ev[4], h->ev[5]);
      t_contract += event_ms(h->ev[5], h->ev[7]);
    }
  } else {
    if (!rows_ordered(h)) { set_error("internal: HODLR rows are not ordered by level"); return BGP_ERR_CUDA; }
    BGP_TRY(h->d_which.reserve(std::max(np, 1), s));
    if (np) BGP_CUDA(cudaMemcpyAsync(h->d_which.p, which, sizeof(unsigned) * np, cudaMemcpyHostToDevice, s));
    BGP_TRY(grad_stream_own_columns(h, np, alpha, c, dg, diag_out ? ddiag : nullptr, &t_solve, &t_contract, ddx.p));
    if (sharded) {  // every shard's partial g, and its rows of diag (and of dx) to every shard
      if (np) BGP_TRY(comm_allreduce_sum_f64(dg, (size_t)np, s));
      if (diag_out) BGP_TRY(exchange_rows(h, ddiag, n, 1, s));
      if (xgrad) BGP_TRY(exchange_rows_wide(h, ddx.p, nd, s));
    }
  }
  if (np && g_out) BGP_CUDA(cudaMemcpyAsync(g_out, dg, sizeof(double) * np, cudaMemcpyDeviceToHost, s));
  if (diag_out) BGP_CUDA(cudaMemcpyAsync(diag_out, ddiag, sizeof(double) * n, cudaMemcpyDeviceToHost, s));
  if (xgrad && dx_out) BGP_CUDA(cudaMemcpyAsync(dx_out, ddx.p, sizeof(double) * n * nd, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  h->grad_t[0] = t_solve;
  h->grad_t[1] = t_contract;
  return BGP_OK;
}

int bgp_hodlr_grad_terms(bgp_hodlr_t* h, const uint32_t* which, const double* r, double* alpha_out, double* g_out,
                         double* diag_out) {
  return hodlr_grad_terms_impl(h, which, r, alpha_out, g_out, diag_out, false, nullptr, "grad_terms");
}

int bgp_hodlr_grad_x_terms(bgp_hodlr_t* h, const uint32_t* which, const double* r, double* alpha_out, double* g_out,
                           double* diag_out, double* dx_out) {
  return hodlr_grad_terms_impl(h, which, r, alpha_out, g_out, diag_out, true, dx_out, "grad_x_terms");
}

// Leave-one-out terms of the HODLR matrix (include/bgp.h), always streamed in the slabs of grad_stream_own_columns:
// pass 1 takes d_j = (K^-1)_jj from each restricted slab solve S = K^-1 E_J; pass 2 (a gradient asked for) solves
// beta = K^-1 (alpha / d), and per slab recomputes S, scales its rows by c and solves T = K^-1 diag(c) S unrestricted
// (diag(c) S is dense), then contracts beta_i alpha_j - T_ij over i in [0, n), j in J (kmat_grad_slab_launch with
// u = beta, v = alpha) and writes diagA_j = alpha_j beta_j - T_jj.
int bgp_hodlr_loo_terms(bgp_hodlr_t* h, const uint32_t* which, const double* r, double* alpha_out, double* d_out,
                        double* beta_out, double* g_out, double* diag_out) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  if (host_exchange(h) || h->opts.shard_count > 1) {
    set_error("loo_terms is not available on a sharded factorisation");
    return BGP_ERR_INVALID;
  }
  const int64_t n = h->n;
  const int np = h->prog.n_params_total;
  if (!rows_ordered(h)) { set_error("internal: HODLR rows are not ordered by level"); return BGP_ERR_CUDA; }
  const bool grad = beta_out || g_out || diag_out;
  if (grad && np > 64) { set_error("gradient supports at most 64 hyper-parameters"); return BGP_ERR_INVALID; }
  cudaStream_t s = h->sA;
  bool forced = false;
  const int64_t c = grad_slab_cols(n, &forced);
  BGP_TRY(h->d_rhs.reserve((size_t)n * 5 + 64, s));
  double* alpha = h->d_rhs.p;
  double* dg = h->d_rhs.p + n;
  double* ddiag = h->d_rhs.p + n + 64;
  double* dd = ddiag + n;
  double* beta = dd + n;  // q = alpha / d, then K^-1 q in place
  double* cw = beta + n;
  BGP_CUDA(cudaMemcpyAsync(alpha, r, sizeof(double) * n, cudaMemcpyHostToDevice, s));
  BGP_TRY(hodlr_solve_dev(h, alpha, 1, n, s, 0));
  BGP_TRY(h->d_inv.reserve((size_t)n * c, s));
  double* W = h->d_inv.p;
  // S = K^-1 E_J for the slab J = [j0, j0 + nc), by the row-restricted solve
  auto slab_solve = [&](int64_t j0, int64_t nc) -> int {
    BGP_CUDA(cudaMemsetAsync(W, 0, sizeof(double) * n * nc, s));
    eye_slab_kernel<<<(unsigned)std::min<int64_t>((nc + 255) / 256, 1184), 256, 0, s>>>(W, n, j0, nc, 0, n);
    BGP_LAUNCH_CHECK();
    return hodlr_solve_dev(h, W, nc, n, s, 0, j0);
  };
  for (int64_t j0 = 0; j0 < n; j0 += c) {
    const int64_t nc = std::min(c, n - j0);
    BGP_TRY(slab_solve(j0, nc));
    BGP_TRY(slab_diag_launch(W, n, j0, nc, dd, s));
  }
  std::vector<double> d_host((size_t)n);
  if (alpha_out) BGP_CUDA(cudaMemcpyAsync(alpha_out, alpha, sizeof(double) * n, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaMemcpyAsync(d_host.data(), dd, sizeof(double) * n, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  if (d_out) memcpy(d_out, d_host.data(), sizeof(double) * n);
  if (!grad) return BGP_OK;
  BGP_TRY(loo_check_diag(d_host.data(), n));
  BGP_TRY(loo_weights_launch(alpha, dd, n, beta, cw, s));
  BGP_TRY(hodlr_solve_dev(h, beta, 1, n, s, 0));
  const int64_t tsize = grad_slab_tile_size(n, np), psize = grad_slab_partial_size(n, c, np);
  BGP_TRY(h->d_gscratch.reserve((size_t)(tsize + psize), s));
  double* tile_part = h->d_gscratch.p;
  double* partial = h->d_gscratch.p + tsize;
  BGP_TRY(h->d_which.reserve(std::max(np, 1), s));
  if (np) BGP_CUDA(cudaMemcpyAsync(h->d_which.p, which, sizeof(unsigned) * np, cudaMemcpyHostToDevice, s));
  for (int64_t j0 = 0; j0 < n; j0 += c) {
    const int64_t nc = std::min(c, n - j0);
    BGP_TRY(slab_solve(j0, nc));
    BGP_TRY(scale_rows_launch(W, n, nc, n, cw, false, s));
    BGP_TRY(hodlr_solve_dev(h, W, nc, n, s, 0));
    BGP_TRY(kmat_grad_slab_launch(h->d_prog.p, h->ndim, np, h->d_which.p, h->d_x.p, n, W, j0, nc, 0, n, beta, alpha,
                                  partial, tile_part, diag_out ? ddiag : nullptr, s));
  }
  BGP_TRY(kmat_grad_slab_finish(np, 0, n, tile_part, dg, s));
  if (beta_out) BGP_CUDA(cudaMemcpyAsync(beta_out, beta, sizeof(double) * n, cudaMemcpyDeviceToHost, s));
  if (np && g_out) BGP_CUDA(cudaMemcpyAsync(g_out, dg, sizeof(double) * np, cudaMemcpyDeviceToHost, s));
  if (diag_out) BGP_CUDA(cudaMemcpyAsync(diag_out, ddiag, sizeof(double) * n, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  return BGP_OK;
}

// One shard's part of the streamed gradient (include/bgp.h): grad_stream_own_columns with the caller's alpha and diag
// (and, with xgrad, its dx rows; a NULL `which` then skips the parameter contraction).
static int hodlr_grad_terms_local_impl(bgp_hodlr* h, const uint32_t* which, const double* alpha_dev,
                                       double* g_part_out, double* diag_dev, bool xgrad, double* dx_dev,
                                       const char* what) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  const int np = (xgrad && !which) ? 0 : h->prog.n_params_total;
  if (np > 64) { set_error("gradient supports at most 64 hyper-parameters"); return BGP_ERR_INVALID; }
  if (xgrad && h->ndim > BGP_MAX_DIM) { set_error("input-coordinate gradients support at most %d dimensions (got %d)", BGP_MAX_DIM, h->ndim); return BGP_ERR_INVALID; }
  if (!alpha_dev) { set_error("%s: alpha_dev is null", what); return BGP_ERR_INVALID; }
  if (xgrad && !dx_dev) { set_error("%s: dx_dev is null", what); return BGP_ERR_INVALID; }
  if (!rows_ordered(h)) { set_error("internal: HODLR rows are not ordered by level"); return BGP_ERR_CUDA; }
  cudaStream_t s = h->sA;
  bool forced = false;
  const int64_t c = grad_slab_cols(h->n, &forced);
  double t_solve = 0, t_contract = 0;
  for (double& t : h->grad_t) t = 0;
  BGP_TRY(h->d_rhs.reserve(64, s));
  double* dg = h->d_rhs.p;
  BGP_TRY(h->d_which.reserve(std::max(np, 1), s));
  if (np) BGP_CUDA(cudaMemcpyAsync(h->d_which.p, which, sizeof(unsigned) * np, cudaMemcpyHostToDevice, s));
  BGP_TRY(grad_stream_own_columns(h, np, alpha_dev, c, dg, diag_dev, &t_solve, &t_contract, xgrad ? dx_dev : nullptr));
  if (np && g_part_out) BGP_CUDA(cudaMemcpyAsync(g_part_out, dg, sizeof(double) * np, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  h->grad_t[0] = t_solve;
  h->grad_t[1] = t_contract;
  return BGP_OK;
}

int bgp_hodlr_grad_terms_local_dev(bgp_hodlr_t* h, const uint32_t* which, const double* alpha_dev, double* g_part_out,
                                   double* diag_dev) {
  return hodlr_grad_terms_local_impl(h, which, alpha_dev, g_part_out, diag_dev, false, nullptr, "grad_terms_local");
}

int bgp_hodlr_grad_x_terms_local_dev(bgp_hodlr_t* h, const uint32_t* which, const double* alpha_dev,
                                     double* g_part_out, double* diag_dev, double* dx_dev) {
  return hodlr_grad_terms_local_impl(h, which, alpha_dev, g_part_out, diag_dev, true, dx_dev, "grad_x_terms_local");
}

// One handle's part of GP.predict's variance / covariance, over its own rows J = [row0, row0 + nloc) ([0, n) unsharded):
//   VAR: out_j = (prior ? k(x*_j, x*_j) : 0) - sum_{i in J} B_ij W_ij                (ns)
//   COV: out   = (prior ? K** : 0) - B[J]^T W[J]          (ns x ns, column-major ld ns: bgp_hodlr_predict's layout)
// with B = K(x, x*) built for the rows J only and W = K^-1 B read in the rows J only, one test-point chunk of c columns
// at a time.  With `grad` (VAR only) each chunk also contracts GP.grad_predict's variance gradient over J:
//   dvar_jq = (prior ? d k(x*_j, x*_j) / d x*_jq : 0) - 2 sum_{i in J} d k(x*_j, x_i) / d x*_jq W_ij   (ns x ndim)
// The chunks, builds and contractions are bgp_hodlr_predict's (and bgp_hodlr_predict_grad's), so on an unsharded handle
// with the prior the result is its bits.  predict_own_prepare validates and reserves without touching the device, so
// that a collective caller can agree on the outcome before anything runs; predict_own_begin then uploads xs and, for
// COV, builds the prior and the resident B[J] (nloc x ns); predict_own_chunk contracts one chunk.
struct PredictOwnRows {
  DevProgram P;
  DevBuf<DevProgram> dprog;
  DevBuf<double> dxs, dB, dkd, dout, ddvar, scratch;
  DevBuf<GemmDesc> ddesc;
  int64_t ns = 0, c = 0;
  int32_t what = 0;
  bool prior = false, grad = false;
};

static int predict_own_prepare(bgp_hodlr* h, const bgp_kernel_spec_t* spec, int64_t ns, int32_t what, bool prior,
                               bool grad, PredictOwnRows* w) {
  if (what != BGP_PREDICT_VAR && what != BGP_PREDICT_COV) { set_error("invalid prediction kind %d", what); return BGP_ERR_INVALID; }
  if (ns < 0) { set_error("negative number of test points"); return BGP_ERR_INVALID; }
  BGP_TRY(build_dev_program(spec, &w->P));
  if (w->P.ndim != h->ndim) { set_error("dimension mismatch: kernel ndim %d, input ndim %d", w->P.ndim, h->ndim); return BGP_ERR_DIM; }
  if (grad && w->P.ndim > BGP_MAX_DIM) { set_error("input-coordinate gradients support at most %d dimensions (got %d)", BGP_MAX_DIM, w->P.ndim); return BGP_ERR_INVALID; }
  w->ns = ns; w->what = what; w->prior = prior; w->grad = grad;
  if (ns == 0) return BGP_OK;
  cudaStream_t s = h->sA;
  const int64_t nloc = h->nloc;
  const int64_t c = std::min(ns, predict_chunk_cols(h->n, 64)), tail = ns - (ns - 1) / c * c;
  w->c = c;
  BGP_TRY(w->dprog.reserve(1, s));
  BGP_TRY(w->dxs.reserve((size_t)ns * h->ndim, s));
  if (what == BGP_PREDICT_VAR) {
    BGP_TRY(w->dB.reserve((size_t)nloc * c, s));
    BGP_TRY(w->dkd.reserve((size_t)c, s));
    BGP_TRY(w->dout.reserve((size_t)ns, s));
    int64_t sc = std::max(predict_var_partial_size(nloc, c), predict_var_partial_size(nloc, tail));
    if (grad) {  // the variance gradient's partials share the scratch with the variance's
      BGP_TRY(w->ddvar.reserve((size_t)ns * h->ndim, s));
      sc = std::max(sc, std::max(x1_grad_partial_size(c, nloc, h->ndim), x1_grad_partial_size(tail, nloc, h->ndim)));
    }
    BGP_TRY(w->scratch.reserve((size_t)sc, s));
  } else {
    BGP_TRY(w->dB.reserve((size_t)nloc * ns, s));
    BGP_TRY(w->dout.reserve((size_t)ns * ns, s));
    // predict_gemm_sub's split-K slices of a full chunk and of the tail; none when the product has one slice
    int64_t nsplit_c, nsplit_t, klen;
    predict_gemm_plan(c, ns, nloc, &nsplit_c, &klen);
    predict_gemm_plan(tail, ns, nloc, &nsplit_t, &klen);
    const int64_t sc = std::max(nsplit_c > 1 ? nsplit_c * c : 0, nsplit_t > 1 ? nsplit_t * tail : 0) * ns;
    if (sc > 0) BGP_TRY(w->scratch.reserve((size_t)sc, s));
    BGP_TRY(w->ddesc.reserve((size_t)std::max(nsplit_c, nsplit_t), s));
  }
  return BGP_OK;
}

static int predict_own_begin(bgp_hodlr* h, PredictOwnRows& w, const double* xs) {
  cudaStream_t s = h->sA;
  BGP_TRY(upload_program(w.P, w.dprog, s));
  BGP_CUDA(cudaMemcpyAsync(w.dxs.p, xs, sizeof(double) * w.ns * h->ndim, cudaMemcpyHostToDevice, s));
  if (w.what == BGP_PREDICT_VAR) {
    if (!w.prior) BGP_CUDA(cudaMemsetAsync(w.dkd.p, 0, sizeof(double) * w.c, s));
    return BGP_OK;
  }
  if (w.prior) BGP_TRY(kmat_symmetric_launch_auto(w.P, w.dprog.p, w.dxs.p, w.ns, nullptr, w.dout.p, w.ns, s));
  else BGP_CUDA(cudaMemsetAsync(w.dout.p, 0, sizeof(double) * w.ns * w.ns, s));
  return kmat_general_launch_auto(w.P, w.dprog.p, w.dxs.p, w.ns, h->d_x.p + h->row0 * h->ndim, h->nloc, w.dB.p,
                                  h->nloc, s);
}

// test points [j0, j0 + nc); Wc: the chunk's first column of W (global row 0), leading dimension ldw
static int predict_own_chunk(bgp_hodlr* h, PredictOwnRows& w, int64_t j0, int64_t nc, const double* Wc, int64_t ldw) {
  cudaStream_t s = h->sA;
  const int64_t nloc = h->nloc;
  if (w.what == BGP_PREDICT_VAR) {
    const double* xc = w.dxs.p + j0 * h->ndim;
    BGP_TRY(kmat_general_launch_auto(w.P, w.dprog.p, xc, nc, h->d_x.p + h->row0 * h->ndim, nloc, w.dB.p, nloc, s));
    if (w.prior) BGP_TRY(kmat_diagonal_launch(w.dprog.p, xc, xc, nc, w.dkd.p, s));
    BGP_TRY(predict_var_launch(w.dB.p, nloc, Wc + h->row0, ldw, nloc, nc, w.dkd.p, w.dout.p + j0, w.scratch, s));
    if (!w.grad) return BGP_OK;
    return kmat_x1_grad_matvec_launch(w.P, w.dprog.p, xc, nc, h->d_x.p + h->row0 * h->ndim, nloc, Wc + h->row0, ldw,
                                      -2.0, w.prior ? 1 : 0, w.ddvar.p + j0 * h->ndim, w.scratch, s);
  }
  // rows j0.. of the column-major result are output COLUMNS j of the row-major one, as in bgp_hodlr_predict
  return predict_gemm_sub(Wc + h->row0, ldw, w.dB.p, nloc, nc, w.ns, nloc, false, w.dout.p + j0, w.ns, w.scratch,
                          w.ddesc, s);
}

// bgp_hodlr_predict and bgp_hodlr_predict_grad on a shard with a matching communicator (include/bgp.h): per test-point
// chunk, this shard's rows of B = K(x, x*) are built into the rows J of an N x c chunk, the collective solve fills the
// other rows from the other shards and runs the top levels, and predict_own_chunk contracts over J; one all-reduce of
// the ns (VAR) or ns^2 (COV) partial results ends it, followed with `grad` by one of the ns x ndim dvar.  The first is
// the prediction's own, so a sharded grad_predict's var has predict's bits.  Every check and reservation comes before
// the first collective, and an all-reduce of a status value turns a failure on any rank into an error on every rank,
// so no rank is left waiting in a later one.
static int hodlr_predict_collective(bgp_hodlr* h, const bgp_kernel_spec_t* spec, const double* xs, int64_t ns,
                                    int32_t what, bool grad, double* out, double* dvar) {
  cudaStream_t s = h->sA;
  const int64_t n = h->n;
  PredictOwnRows w;
  DevBuf<double> dW;
  int st = predict_own_prepare(h, spec, ns, what, h->opts.shard_rank == 0, grad, &w);
  if (st == BGP_OK && ns == 0) return BGP_OK;  // ns is replicated: every rank returns here
  if (st == BGP_OK) st = dW.alloc((size_t)n * w.c, s);
  if (st == BGP_OK) {  // exchange_rows' staging for the solve's 64-column groups
    int64_t rows_pad = 0;
    for (int64_t r : h->shard_rows) rows_pad = std::max(rows_pad, r);
    st = h->d_xsend.reserve((size_t)64 * rows_pad, s);
    if (st == BGP_OK) st = h->d_xrecv.reserve((size_t)64 * rows_pad * h->opts.shard_count, s);
  }
  double failed = st == BGP_OK ? 0.0 : 1.0;
  BGP_CUDA(cudaMemcpyAsync(h->d_scalar.p, &failed, sizeof(double), cudaMemcpyHostToDevice, s));
  BGP_TRY(comm_allreduce_sum_f64(h->d_scalar.p, 1, s));
  BGP_CUDA(cudaMemcpyAsync(&failed, h->d_scalar.p, sizeof(double), cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  if (st != BGP_OK) return st;
  if (failed != 0.0) {
    set_error("predict: %d other shard(s) could not validate or reserve their part", (int)failed);
    return BGP_ERR_NOMEM;
  }
  BGP_TRY(predict_own_begin(h, w, xs));
  const int nd = h->ndim;
  for (int64_t j0 = 0; j0 < ns; j0 += w.c) {
    const int64_t nc = std::min(w.c, ns - j0);
    BGP_TRY(kmat_general_launch_auto(w.P, w.dprog.p, w.dxs.p + j0 * nd, nc, h->d_x.p + h->row0 * nd, h->nloc,
                                     dW.p + h->row0, n, s));
    BGP_TRY(hodlr_solve_dev(h, dW.p, nc, n, s, 0));
    BGP_TRY(predict_own_chunk(h, w, j0, nc, dW.p, n));
  }
  const size_t count = (size_t)(what == BGP_PREDICT_VAR ? ns : ns * ns);
  BGP_TRY(comm_allreduce_sum_f64(w.dout.p, count, s));
  BGP_CUDA(cudaMemcpyAsync(out, w.dout.p, sizeof(double) * count, cudaMemcpyDeviceToHost, s));
  if (grad) {
    BGP_TRY(comm_allreduce_sum_f64(w.ddvar.p, (size_t)(ns * nd), s));
    BGP_CUDA(cudaMemcpyAsync(dvar, w.ddvar.p, sizeof(double) * ns * nd, cudaMemcpyDeviceToHost, s));
  }
  BGP_CUDA(cudaStreamSynchronize(s));
  return BGP_OK;
}

// One handle's part of the prediction (and with `grad` its variance gradient into dvar) from the caller's solved W
// (include/bgp.h).  Issues no collective.
static int hodlr_predict_local(bgp_hodlr* h, const bgp_kernel_spec_t* spec, const double* xs, int64_t ns, int32_t what,
                               bool grad, const double* w_dev, int64_t ldw, int32_t add_prior, double* out,
                               double* dvar) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  if (ns > 0 && !w_dev) { set_error("predict_local: w_dev is null"); return BGP_ERR_INVALID; }
  if (ldw < h->n) { set_error("predict_local: ldw %lld < n %lld", (long long)ldw, (long long)h->n); return BGP_ERR_INVALID; }
  PredictOwnRows w;
  BGP_TRY(predict_own_prepare(h, spec, ns, what, add_prior != 0, grad, &w));
  if (ns == 0) return BGP_OK;
  cudaStream_t s = h->sA;
  BGP_TRY(predict_own_begin(h, w, xs));
  for (int64_t j0 = 0; j0 < ns; j0 += w.c)
    BGP_TRY(predict_own_chunk(h, w, j0, std::min(w.c, ns - j0), w_dev + j0 * ldw, ldw));
  const size_t count = (size_t)(what == BGP_PREDICT_VAR ? ns : ns * ns);
  BGP_CUDA(cudaMemcpyAsync(out, w.dout.p, sizeof(double) * count, cudaMemcpyDeviceToHost, s));
  if (grad) BGP_CUDA(cudaMemcpyAsync(dvar, w.ddvar.p, sizeof(double) * ns * h->ndim, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  return BGP_OK;
}

int bgp_hodlr_predict_local_dev(bgp_hodlr_t* h, const bgp_kernel_spec_t* spec, const double* xs, int64_t ns,
                                int32_t what, const double* w_dev, int64_t ldw, int32_t add_prior, double* out) {
  return hodlr_predict_local(h, spec, xs, ns, what, false, w_dev, ldw, add_prior, out, nullptr);
}

int bgp_hodlr_predict_grad_local_dev(bgp_hodlr_t* h, const bgp_kernel_spec_t* spec, const double* xs, int64_t ns,
                                     const double* w_dev, int64_t ldw, int32_t add_prior, double* var, double* dvar) {
  return hodlr_predict_local(h, spec, xs, ns, BGP_PREDICT_VAR, true, w_dev, ldw, add_prior, var, dvar);
}

// GP.predict's covariance on an unsharded handle into dC (ns x ns on the device, allocated here; row-major as
// bgp_hodlr_predict returns it): B = K(x, x*) stays resident (n*ns), W one chunk (n*c): C[:, chunk] = K**[:, chunk] -
// B^T W_chunk, in the reference's orientation (K_h^-1 is symmetric only to tol).  P is the validated program of the
// prediction's kernel.  bgp_hodlr_predict copies dC out; bgp_hodlr_sample draws from it on the device.
static int hodlr_predict_cov_dev(bgp_hodlr* h, const DevProgram& P, const double* xs, int64_t ns, DevBuf<double>& dC) {
  const int64_t n = h->n;
  const int nd = h->ndim;
  cudaStream_t s = h->sA;
  DevBuf<DevProgram> dprog;
  DevBuf<double> dxs, dB, dW, scratch;
  DevBuf<GemmDesc> ddesc;
  BGP_TRY(upload_program(P, dprog, s));
  const int64_t c = std::min(ns, predict_chunk_cols(n, 64));
  BGP_TRY(dW.alloc((size_t)n * c, s));
  BGP_TRY(dxs.alloc((size_t)ns * nd, s));
  BGP_TRY(dB.alloc((size_t)n * ns, s));
  BGP_TRY(dC.alloc((size_t)ns * ns, s));
  BGP_CUDA(cudaMemcpyAsync(dxs.p, xs, sizeof(double) * ns * nd, cudaMemcpyHostToDevice, s));
  BGP_TRY(kmat_symmetric_launch_auto(P, dprog.p, dxs.p, ns, nullptr, dC.p, ns, s));
  BGP_TRY(kmat_general_launch_auto(P, dprog.p, dxs.p, ns, h->d_x.p, n, dB.p, n, s));
  for (int64_t j0 = 0; j0 < ns; j0 += c) {
    const int64_t nc = std::min(c, ns - j0);
    BGP_CUDA(cudaMemcpyAsync(dW.p, dB.p + j0 * n, sizeof(double) * n * nc, cudaMemcpyDeviceToDevice, s));
    BGP_TRY(hodlr_solve_dev(h, dW.p, nc, n, s, 0));
    // column-major C (ld ns): rows j0.. of the chunk are output COLUMNS j of the row-major result
    BGP_TRY(predict_gemm_sub(dW.p, n, dB.p, n, nc, ns, n, false, dC.p + j0, ns, scratch, ddesc, s));
  }
  return BGP_OK;
}

// GP.predict's variance / covariance on the stored factorisation.  The test points are streamed in chunks of a multiple
// of 64 columns, so W = K^-1 B is solved in the same 64-column groups as apply_inverse and matches it bit for bit.
// On a shard with a matching communicator the call is collective (hodlr_predict_collective).
int bgp_hodlr_predict(bgp_hodlr_t* h, const bgp_kernel_spec_t* spec, const double* xs, int64_t ns, int32_t what,
                      double* out) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  if (host_exchange(h)) { set_error("predict is not available on a sharded factorisation"); return BGP_ERR_INVALID; }
  if (h->opts.shard_count > 1) return hodlr_predict_collective(h, spec, xs, ns, what, false, out, nullptr);
  if (what != BGP_PREDICT_VAR && what != BGP_PREDICT_COV) { set_error("invalid prediction kind %d", what); return BGP_ERR_INVALID; }
  if (ns < 0) { set_error("negative number of test points"); return BGP_ERR_INVALID; }
  DevProgram P;
  BGP_TRY(build_dev_program(spec, &P));
  if (P.ndim != h->ndim) { set_error("dimension mismatch: kernel ndim %d, input ndim %d", P.ndim, h->ndim); return BGP_ERR_DIM; }
  if (ns == 0) return BGP_OK;
  const int64_t n = h->n;
  const int nd = h->ndim;
  cudaStream_t s = h->sA;
  DevBuf<DevProgram> dprog;
  DevBuf<double> dxs, dB, dW, dkd, dvar, dC, scratch;
  if (what == BGP_PREDICT_VAR) {
    BGP_TRY(upload_program(P, dprog, s));
    const int64_t c = std::min(ns, predict_chunk_cols(n, 64));
    BGP_TRY(dW.alloc((size_t)n * c, s));
    // workspace 2*n*c + O(c): var_j = k(x*_j, x*_j) - B_j . (K^-1 B)_j, chunk by chunk
    BGP_TRY(dxs.alloc((size_t)c * nd, s));
    BGP_TRY(dB.alloc((size_t)n * c, s));
    BGP_TRY(dkd.alloc((size_t)c, s));
    BGP_TRY(dvar.alloc((size_t)c, s));
    for (int64_t j0 = 0; j0 < ns; j0 += c) {
      const int64_t nc = std::min(c, ns - j0);
      BGP_CUDA(cudaMemcpyAsync(dxs.p, xs + j0 * nd, sizeof(double) * nc * nd, cudaMemcpyHostToDevice, s));
      BGP_TRY(kmat_general_launch_auto(P, dprog.p, dxs.p, nc, h->d_x.p, n, dB.p, n, s));
      BGP_CUDA(cudaMemcpyAsync(dW.p, dB.p, sizeof(double) * n * nc, cudaMemcpyDeviceToDevice, s));
      BGP_TRY(hodlr_solve_dev(h, dW.p, nc, n, s, 0));
      BGP_TRY(kmat_diagonal_launch(dprog.p, dxs.p, dxs.p, nc, dkd.p, s));
      BGP_TRY(predict_var_launch(dB.p, n, dW.p, n, n, nc, dkd.p, dvar.p, scratch, s));
      BGP_CUDA(cudaMemcpyAsync(out + j0, dvar.p, sizeof(double) * nc, cudaMemcpyDeviceToHost, s));
    }
  } else {
    BGP_TRY(hodlr_predict_cov_dev(h, P, xs, ns, dC));
    BGP_CUDA(cudaMemcpyAsync(out, dC.p, sizeof(double) * ns * ns, cudaMemcpyDeviceToHost, s));
  }
  BGP_CUDA(cudaStreamSynchronize(s));
  return BGP_OK;
}

// GP.grad_predict's var and dvar: bgp_hodlr_predict's VAR chunks, whose W is already K_h^-1 K(x, x*_chunk), then
// dvar = dprior - 2 sum_j d1 k(x*, x_j) W_j (kmat_x1_grad_matvec_launch).  On a shard with a matching communicator the
// call is collective (hodlr_predict_collective).
int bgp_hodlr_predict_grad(bgp_hodlr_t* h, const bgp_kernel_spec_t* spec, const double* xs, int64_t ns, double* var,
                           double* dvar) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  if (host_exchange(h)) { set_error("predict_grad is not available on a sharded factorisation"); return BGP_ERR_INVALID; }
  if (h->opts.shard_count > 1) return hodlr_predict_collective(h, spec, xs, ns, BGP_PREDICT_VAR, true, var, dvar);
  if (ns < 0) { set_error("negative number of test points"); return BGP_ERR_INVALID; }
  DevProgram P;
  BGP_TRY(build_dev_program(spec, &P));
  if (P.ndim != h->ndim) { set_error("dimension mismatch: kernel ndim %d, input ndim %d", P.ndim, h->ndim); return BGP_ERR_DIM; }
  if (P.ndim > BGP_MAX_DIM) { set_error("input-coordinate gradients support at most %d dimensions (got %d)", BGP_MAX_DIM, P.ndim); return BGP_ERR_INVALID; }
  if (ns == 0) return BGP_OK;
  const int64_t n = h->n;
  const int nd = h->ndim;
  cudaStream_t s = h->sA;
  DevBuf<DevProgram> dprog;
  DevBuf<double> dxs, dB, dW, dkd, dvar_c, ddvar, scratch;
  BGP_TRY(upload_program(P, dprog, s));
  const int64_t c = std::min(ns, predict_chunk_cols(n, 64));
  // workspace 2*n*c + O(c * ndim): bgp_hodlr_predict's VAR workspace plus the chunk's dvar
  BGP_TRY(dW.alloc((size_t)n * c, s));
  BGP_TRY(dxs.alloc((size_t)c * nd, s));
  BGP_TRY(dB.alloc((size_t)n * c, s));
  BGP_TRY(dkd.alloc((size_t)c, s));
  BGP_TRY(dvar_c.alloc((size_t)c, s));
  BGP_TRY(ddvar.alloc((size_t)c * nd, s));
  for (int64_t j0 = 0; j0 < ns; j0 += c) {
    const int64_t nc = std::min(c, ns - j0);
    // the steps of bgp_hodlr_predict's VAR loop
    BGP_CUDA(cudaMemcpyAsync(dxs.p, xs + j0 * nd, sizeof(double) * nc * nd, cudaMemcpyHostToDevice, s));
    BGP_TRY(kmat_general_launch_auto(P, dprog.p, dxs.p, nc, h->d_x.p, n, dB.p, n, s));
    BGP_CUDA(cudaMemcpyAsync(dW.p, dB.p, sizeof(double) * n * nc, cudaMemcpyDeviceToDevice, s));
    BGP_TRY(hodlr_solve_dev(h, dW.p, nc, n, s, 0));
    BGP_TRY(kmat_diagonal_launch(dprog.p, dxs.p, dxs.p, nc, dkd.p, s));
    BGP_TRY(predict_var_launch(dB.p, n, dW.p, n, n, nc, dkd.p, dvar_c.p, scratch, s));
    BGP_CUDA(cudaMemcpyAsync(var + j0, dvar_c.p, sizeof(double) * nc, cudaMemcpyDeviceToHost, s));
    BGP_TRY(kmat_x1_grad_matvec_launch(P, dprog.p, dxs.p, nc, h->d_x.p, n, dW.p, n, -2.0, 1, ddvar.p, scratch, s));
    BGP_CUDA(cudaMemcpyAsync(dvar + j0 * nd, ddvar.p, sizeof(double) * nc * nd, cudaMemcpyDeviceToHost, s));
  }
  BGP_CUDA(cudaStreamSynchronize(s));
  return BGP_OK;
}

// bgp_hodlr_predict's covariance drawn from on the device (include/bgp.h); unsharded handles only
int bgp_hodlr_sample(bgp_hodlr_t* h, const bgp_kernel_spec_t* spec, const double* xs, int64_t ns, const double* mean,
                     const double* z, int64_t size, double jitter, double* out) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  if (h->opts.shard_count > 1) { set_error("sample is not available on a sharded factorisation"); return BGP_ERR_INVALID; }
  BGP_TRY(mvn_sample_check(ns, size, jitter));
  DevProgram P;
  BGP_TRY(build_dev_program(spec, &P));
  if (P.ndim != h->ndim) { set_error("dimension mismatch: kernel ndim %d, input ndim %d", P.ndim, h->ndim); return BGP_ERR_DIM; }
  if (ns == 0 || size == 0) return BGP_OK;
  DevBuf<double> dC;
  BGP_TRY(sample_mark(0, h->sA));
  BGP_TRY(hodlr_predict_cov_dev(h, P, xs, ns, dC));
  return mvn_draw_host_io(dC.p, ns, mean, z, size, jitter, out, h->sA);
}

// ---- symmetric factor K~ = W W^T (hodlr_sym.cu) ------------------------------------------------------------------
// Built from the leaves' L D L^T and the raw ACA factors (the V panels), which compute() leaves untouched after it ends,
// on the first call that needs it after a compute(); compute() marks it stale.  On a shard the factor splits at the
// shard cut like compute() (DESIGN.md §5): the leaves and owned levels on this shard's rows, one all-gather of this
// shard's rows of the top levels' columns, then the top levels on every shard.  With a matching communicator
// bgp_hodlr_sym_factor does all of it collectively; a host-exchange shard runs the steps one by one
// (bgp_hodlr_sym_factor_local, _export_top, _import_top, _finish_top).

// this handle's levels, nodes and leaves for sym_prepare
static int sym_prepare_handle(bgp_hodlr* h, bool staging) {
  if (!h->sym && !(h->sym = sym_create())) { set_error("out of host memory"); return BGP_ERR_NOMEM; }
  const int nlev = (int)h->levels.size();
  std::vector<int> lev, nodes;
  for (const LevelInfo& L : h->levels) {
    lev.insert(lev.end(), {L.r, L.ucol, L.vcol, (int)L.nodes.size()});
    for (int id : L.nodes) {
      const HNode& nd = h->nodes[id];
      nodes.insert(nodes.end(), {nd.start, nd.size, nd.half, nd.rank, id});
    }
  }
  std::vector<int64_t> leaves;
  int64_t off = 0;
  for (int id : h->leaves) {  // d_L's layout (hodlr_compute_dev_impl); ncols: the leaf's local ancestor columns
    const HNode& nd = h->nodes[id];
    const int ncols = nd.depth < nlev ? h->levels[nd.depth].ucol : h->loc.ucols;
    leaves.insert(leaves.end(), {(int64_t)nd.start, (int64_t)nd.size, (int64_t)ncols, off});
    off += (int64_t)nd.size * nd.size;
  }
  const int cut = h->opts.shard_count > 1 ? std::min(h->cut_depth, nlev) : 0;
  return sym_prepare(h->sym, h->n, h->row0, h->nloc, cut, nlev, lev.data(), nodes.data(), (int)h->leaves.size(),
                     leaves.data(), h->max_leaf, h->d_L.p, staging, h->sA);
}

static int sym_local_handle(bgp_hodlr* h) {
  return sym_build_local(h->sym, h->top.vbase(), h->loc.vbase(), h->loc.ld, h->sA);
}

// One all-reduce of one double over the shards: each failing shard adds 2^rank.  *failed_shard = the highest failing
// shard, or -1 when none failed.
static int allreduce_failed_shard(bgp_hodlr* h, bool failed, int* failed_shard) {
  cudaStream_t s = h->sA;
  double v = failed ? std::ldexp(1.0, h->opts.shard_rank) : 0.0;
  BGP_CUDA(cudaMemcpyAsync(h->d_scalar.p, &v, sizeof(double), cudaMemcpyHostToDevice, s));
  BGP_TRY(comm_allreduce_sum_f64(h->d_scalar.p, 1, s));
  BGP_CUDA(cudaMemcpyAsync(&v, h->d_scalar.p, sizeof(double), cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  *failed_shard = v > 0.0 ? std::ilogb(v) : -1;
  return BGP_OK;
}

// bgp_hodlr_sym_factor on a shard with a matching communicator.  Every check and reservation comes first, then an
// all-reduce of a status; the local build, then a second one, so that a shard whose leaf or node has no factor makes
// every rank return before the all-gather instead of leaving the others waiting in it; the all-gather of this shard's
// rows of the top columns, the top levels, and one all-reduce of the partial log-determinants.
static int sym_build_collective(bgp_hodlr* h) {
  cudaStream_t s = h->sA;
  int64_t rows_pad = 0, rtop = 0;
  for (int64_t r : h->shard_rows) rows_pad = std::max(rows_pad, r);
  int st = sym_prepare_handle(h, true);
  if (st == BGP_OK) {  // exchange_rows' staging for the top columns and for the apply's 64-column groups
    sym_top_panel(h->sym, &rtop);
    const size_t per = (size_t)std::max<int64_t>(rtop, 64) * rows_pad;
    st = h->d_xsend.reserve(per, s);
    if (st == BGP_OK) st = h->d_xrecv.reserve(per * h->opts.shard_count, s);
  }
  int failed = -1;
  BGP_TRY(allreduce_failed_shard(h, st != BGP_OK, &failed));
  if (st != BGP_OK) return st;
  if (failed >= 0) {
    set_error("the symmetric factor: shard %d of %d could not validate or reserve its part", failed,
              h->opts.shard_count);
    return BGP_ERR_INVALID;
  }
  st = sym_local_handle(h);
  BGP_TRY(allreduce_failed_shard(h, st != BGP_OK, &failed));
  if (st != BGP_OK) return st;
  if (failed >= 0) {
    set_error("the HODLR matrix has no symmetric factor: the local part failed on shard %d of %d (that shard names the "
              "leaf or node)", failed, h->opts.shard_count);
    return BGP_ERR_LINALG;
  }
  double* ptop = sym_top_panel(h->sym, &rtop);
  BGP_TRY(exchange_rows(h, ptop, h->n, rtop, s));
  double ld = 0.0;
  BGP_TRY(sym_build_top(h->sym, h->opts.shard_rank == 0, s, &ld));  // the same launches and data on every shard
  BGP_CUDA(cudaMemcpyAsync(h->d_scalar.p, &ld, sizeof(double), cudaMemcpyHostToDevice, s));
  BGP_TRY(comm_allreduce_sum_f64(h->d_scalar.p, 1, s));
  BGP_CUDA(cudaMemcpyAsync(&ld, h->d_scalar.p, sizeof(double), cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  h->sym_log_det = ld;
  return BGP_OK;
}

static int sym_require(bgp_hodlr* h, const char* what) {
  if (h && host_exchange(h)) {
    set_error("%s is not available on a host-exchange shard of a sharded factorisation (shard %d of %d without a "
              "matching communicator): use bgp_hodlr_sym_factor_local / _export_top / _import_top / _finish_top and "
              "bgp_hodlr_sym_apply_local_dev / _top_dev", what, h->opts.shard_rank, h->opts.shard_count);
    return BGP_ERR_INVALID;
  }
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  if (h->sym_current) return BGP_OK;
  BGP_TRY(require_device());
  h->sym_stage = 0;
  if (h->opts.shard_count > 1) {
    BGP_TRY(sym_build_collective(h));
  } else {
    BGP_TRY(sym_prepare_handle(h, false));
    BGP_TRY(sym_local_handle(h));
    BGP_TRY(sym_build_top(h->sym, 1, h->sA, &h->sym_log_det));
  }
  h->sym_current = true;
  return BGP_OK;
}

int bgp_hodlr_sym_factor(bgp_hodlr_t* h) { return sym_require(h, "the symmetric factor"); }

// On a shard with a matching communicator: collective, z replicated, the result replicated (each 64-column group's own
// rows all-gathered between the local and the top levels).
int bgp_hodlr_sym_apply(bgp_hodlr_t* h, double* z, int64_t nrhs, int64_t ldz, int32_t transpose) {
  BGP_TRY(sym_require(h, "the symmetric factor"));
  if (nrhs <= 0) return BGP_OK;
  if (ldz < h->n) { set_error("dimension mismatch: ldz < n"); return BGP_ERR_DIM; }
  std::function<int(double*, int)> exchange;
  if (h->opts.shard_count > 1) exchange = [h](double* Z, int nc) { return exchange_rows(h, Z, h->n, nc, h->sA); };
  return sym_apply(h->sym, z, nrhs, ldz, transpose ? 1 : 0, h->sA, exchange);
}

int bgp_hodlr_sym_log_determinant(bgp_hodlr_t* h, double* out) {
  BGP_TRY(sym_require(h, "the symmetric factor"));
  *out = h->sym_log_det;
  return BGP_OK;
}

int bgp_hodlr_sym_last_timing(const bgp_hodlr_t* h, double* ms2) {
  if (!h) { set_error("null handle"); return BGP_ERR_INVALID; }
  ms2[0] = ms2[1] = 0.0;
  if (h->sym) sym_timing(h->sym, ms2);
  return BGP_OK;
}

int bgp_selftest_hodlr_sym_orthogonality(bgp_hodlr_t* h, double* out) {
  BGP_TRY(sym_require(h, "the symmetric factor"));
  return sym_orthogonality(h->sym, out, h->sA);
}

int bgp_selftest_hodlr_sym_householder_nodes(bgp_hodlr_t* h, int32_t* counts, int32_t cap, int32_t* nlev) {
  BGP_TRY(sym_require(h, "the symmetric factor"));
  *nlev = sym_householder_nodes(h->sym, counts, cap);
  return BGP_OK;
}

int bgp_hodlr_num_nodes(const bgp_hodlr_t* h, int64_t* out) {
  if (!h) { set_error("null handle"); return BGP_ERR_INVALID; }
  *out = (int64_t)h->nodes.size();
  return BGP_OK;
}

int bgp_hodlr_node_info(const bgp_hodlr_t* h, bgp_hodlr_node_info_t* out) {
  if (!h) { set_error("null handle"); return BGP_ERR_INVALID; }
  for (size_t i = 0; i < h->nodes.size(); ++i) {
    const HNode& nd = h->nodes[i];
    out[i].start = nd.start; out[i].size = nd.size; out[i].half = nd.half; out[i].is_leaf = nd.is_leaf;
    out[i].parent = nd.parent; out[i].direction = nd.dir; out[i].depth = nd.depth; out[i].rank = nd.rank;
    out[i].rng_draws = nd.draws; out[i].dense_fallback = nd.fallback;
  }
  return BGP_OK;
}

int bgp_hodlr_node_pivots(const bgp_hodlr_t* hc, int64_t node, int32_t* rows, int32_t* cols) {
  bgp_hodlr_t* h = const_cast<bgp_hodlr_t*>(hc);
  if (!h || node < 0 || node >= (int64_t)h->nodes.size()) { set_error("node index out of range"); return BGP_ERR_INDEX; }
  const HNode& nd = h->nodes[node];
  // dense fallback nodes (exhaust_mode = dense) have no pivot list: their factors are the identity / the block itself
  if (nd.is_leaf || h->piv_off[node] < 0 || nd.rank == 0 ||
      (nd.fallback && h->opts.exhaust_mode == BGP_EXHAUST_DENSE))
    return BGP_OK;
  BGP_CUDA(cudaMemcpy(rows, h->d_piv_rows.p + h->piv_off[node], sizeof(int) * nd.rank, cudaMemcpyDeviceToHost));
  BGP_CUDA(cudaMemcpy(cols, h->d_piv_cols.p + h->piv_off[node], sizeof(int) * nd.rank, cudaMemcpyDeviceToHost));
  return BGP_OK;
}

// The node's columns [vcol, vcol + rank) of its level's V panel, rows [start, start + size): the up-sweep reads this
// panel but never writes it (the U panel is the copy it solves in place), so these are the ACA's factors as it left them.
int bgp_hodlr_node_factors(const bgp_hodlr_t* h, int64_t node, double* out) {
  if (!h) { set_error("null handle"); return BGP_ERR_INVALID; }
  if (!h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  if (h->opts.shard_count > 1) { set_error("node factors are not available on a sharded factorisation"); return BGP_ERR_INVALID; }
  if (node < 0 || node >= (int64_t)h->nodes.size() || h->nodes[node].is_leaf) {
    set_error("node %lld is not an internal node", (long long)node);
    return BGP_ERR_INDEX;
  }
  const HNode& nd = h->nodes[node];
  if (nd.rank == 0) return BGP_OK;
  const LevelInfo& L = h->levels[nd.depth];
  const PanelSet& ps = h->pset(L);
  const double* src = ps.vbase() + (int64_t)L.vcol * ps.ld + nd.start;
  BGP_CUDA(cudaMemcpy2D(out, sizeof(double) * nd.size, src, sizeof(double) * ps.ld, sizeof(double) * nd.size, nd.rank,
                        cudaMemcpyDeviceToHost));
  return BGP_OK;
}

int bgp_hodlr_last_draw_paths(const bgp_hodlr_t* h, uint64_t* out4) {
  if (!h) { set_error("null handle"); return BGP_ERR_INVALID; }
  if (!h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  for (int i = 0; i < 4; ++i) out4[i] = h->draw_paths[i];
  return BGP_OK;
}

int bgp_hodlr_last_eval_units(const bgp_hodlr_t* h, uint64_t* out2) {
  if (!h) { set_error("null handle"); return BGP_ERR_INVALID; }
  if (!h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  for (int i = 0; i < 2; ++i) out2[i] = h->eval_units[i];
  return BGP_OK;
}

int bgp_hodlr_last_timing(const bgp_hodlr_t* h, double* ms5) {
  if (!h) { set_error("null handle"); return BGP_ERR_INVALID; }
  for (int i = 0; i < 5; ++i) ms5[i] = h->t_ms[i];
  return BGP_OK;
}
int bgp_hodlr_last_grad_timing(const bgp_hodlr_t* h, double* out4) {
  if (!h) { set_error("null handle"); return BGP_ERR_INVALID; }
  for (int i = 0; i < 4; ++i) out4[i] = h->grad_t[i];
  return BGP_OK;
}
int bgp_hodlr_set_profiling(bgp_hodlr_t* h, int on) {
  if (!h) { set_error("null handle"); return BGP_ERR_INVALID; }
  h->profile = on != 0;
  return BGP_OK;
}
int bgp_hodlr_last_aca_profile(const bgp_hodlr_t* h, double* p12) {
  if (!h) { set_error("null handle"); return BGP_ERR_INVALID; }
  for (int i = 0; i < 12; ++i) p12[i] = h->prof[i];
  return BGP_OK;
}
int bgp_hodlr_last_work(const bgp_hodlr_t* h, double* w6) {
  if (!h) { set_error("null handle"); return BGP_ERR_INVALID; }
  for (int i = 0; i < 6; ++i) w6[i] = h->work[i];
  return BGP_OK;
}

// ---- diagnostics: the dense building blocks of the big-rank path, callable on their own (tests/test_gpu_linalg.py) ----
int bgp_selftest_lu(int32_t n, int32_t nrhs, const double* S_host, double* R_host, double* logdet) {
  BGP_TRY(require_device());
  if (n <= 0 || nrhs < 0) { set_error("bgp_selftest_lu: bad sizes"); return BGP_ERR_INVALID; }
  cudaStream_t s = 0;
  DevBuf<double> dS, dR, dld;
  LuWorkspace ws;
  BGP_TRY(dS.alloc((size_t)n * n + n, s));
  BGP_TRY(dR.alloc(std::max<size_t>((size_t)n * nrhs, 1), s));
  BGP_TRY(dld.alloc(1, s));
  BGP_CUDA(cudaMemcpyAsync(dS.p, S_host, sizeof(double) * n * n, cudaMemcpyHostToDevice, s));
  if (nrhs) BGP_CUDA(cudaMemcpyAsync(dR.p, R_host, sizeof(double) * n * nrhs, cudaMemcpyHostToDevice, s));
  std::vector<LuNode> nodes(1);
  nodes[0].S = dS.p; nodes[0].piv = reinterpret_cast<int*>(dS.p + (size_t)n * n); nodes[0].logdet = dld.p;
  BGP_TRY(lu_factor_batch(ws, nodes, n, s));
  BGP_TRY(lu_solve_batch(ws, nodes, n, dR.p, 0, n, nrhs, false, s));
  if (nrhs) BGP_CUDA(cudaMemcpyAsync(R_host, dR.p, sizeof(double) * n * nrhs, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaMemcpyAsync(logdet, dld.p, sizeof(double), cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  return BGP_OK;
}

int bgp_selftest_gemm(int32_t a_kcontig, int32_t b_kcontig, int32_t m, int32_t n, int32_t k, const double* A_host,
                      int64_t lda, const double* B_host, int64_t ldb, double* C_host, int64_t ldc, int32_t mode) {
  BGP_TRY(require_device());
  if (m <= 0 || n <= 0 || k <= 0) { set_error("bgp_selftest_gemm: bad sizes"); return BGP_ERR_INVALID; }
  if (mode & ~(GD_ATOMIC_ADD | GD_LOWER)) { set_error("bgp_selftest_gemm: bad mode %d", mode); return BGP_ERR_INVALID; }
  cudaStream_t s = 0;
  const size_t na = (size_t)(a_kcontig ? m : k) * lda, nb = (size_t)(b_kcontig ? n : k) * ldb, nc = (size_t)n * ldc;
  DevBuf<double> dA, dB, dC;
  DevBuf<GemmDesc> dd;
  BGP_TRY(dA.alloc(na, s)); BGP_TRY(dB.alloc(nb, s)); BGP_TRY(dC.alloc(nc, s)); BGP_TRY(dd.alloc(1, s));
  BGP_CUDA(cudaMemcpyAsync(dA.p, A_host, sizeof(double) * na, cudaMemcpyHostToDevice, s));
  BGP_CUDA(cudaMemcpyAsync(dB.p, B_host, sizeof(double) * nb, cudaMemcpyHostToDevice, s));
  BGP_CUDA(cudaMemcpyAsync(dC.p, C_host, sizeof(double) * nc, cudaMemcpyHostToDevice, s));
  GemmDesc g;
  g.A = dA.p; g.B = dB.p; g.C = dC.p; g.M = m; g.N = n; g.K = k; g.mode = mode;
  g.lda = lda; g.ldb = ldb; g.ldc = ldc;
  BGP_CUDA(cudaMemcpyAsync(dd.p, &g, sizeof(g), cudaMemcpyHostToDevice, s));
  if (a_kcontig && b_kcontig) BGP_TRY((gemm_dmma_launch<true, true>(dd.p, 1, m, n, nullptr, s)));
  else if (a_kcontig) BGP_TRY((gemm_dmma_launch<true, false>(dd.p, 1, m, n, nullptr, s)));
  else if (b_kcontig) BGP_TRY((gemm_dmma_launch<false, true>(dd.p, 1, m, n, nullptr, s)));
  else BGP_TRY((gemm_dmma_launch<false, false>(dd.p, 1, m, n, nullptr, s)));
  BGP_CUDA(cudaMemcpyAsync(C_host, dC.p, sizeof(double) * nc, cudaMemcpyDeviceToHost, s));
  BGP_CUDA(cudaStreamSynchronize(s));
  return BGP_OK;
}

// ---- multi-GPU exchange (SURVEY.md §8e) -----------------------------------------------------------------------
int bgp_hodlr_top_panel(bgp_hodlr_t* h, double** ptr_dev, int64_t* row0, int64_t* rows, int64_t* cols, int64_t* ld) {
  if (!h) { set_error("null handle"); return BGP_ERR_INVALID; }
  const int cut = std::min<int>(h->cut_depth, (int)h->levels.size());
  *ptr_dev = h->top.U.p;
  *row0 = h->row0; *rows = h->nloc;
  (void)cut;
  *cols = h->top.ucols;
  *ld = h->n;
  return BGP_OK;
}


int bgp_hodlr_shard_rows(const bgp_hodlr_t* h, int32_t s, int64_t* row0, int64_t* rows) {
  if (!h || s < 0 || s >= (int)h->shard_rows.size()) { set_error("shard index out of range"); return BGP_ERR_INDEX; }
  *row0 = h->shard_row0[s]; *rows = h->shard_rows[s];
  return BGP_OK;
}

// export / import / finish_top belong between a host-exchange compute and its (one) finish_top: finish_top updates the
// top panel in place, so a second one, or an import after it, would work on rows that were already finished.
static int require_top_pending(const bgp_hodlr* h, const char* what) {
  if (h->top_pending) return BGP_OK;
  if (!h->computed) {
    set_error("%s: no sharded factorisation is waiting for its top levels (the solver has not been computed)", what);
    return BGP_ERR_NOT_COMPUTED;
  }
  set_error("%s: the factorisation is complete (unsharded, or finish_top was already called)", what);
  return BGP_ERR_INVALID;
}

int bgp_hodlr_export_top(bgp_hodlr_t* h, double* buf_dev, int64_t rows_pad) {
  if (!h) { set_error("null handle"); return BGP_ERR_INVALID; }
  BGP_TRY(require_top_pending(h, "export_top"));
  if (rows_pad < h->nloc) {  // checked even when there is nothing to pack, as import_top does
    set_error("rows_pad %lld smaller than this shard (%lld rows)", (long long)rows_pad, (long long)h->nloc);
    return BGP_ERR_INVALID;
  }
  const int64_t cols = top_cols(h);
  if (cols == 0 || h->nloc == 0) return BGP_OK;
  pack_rows_kernel<<<1184, 256, 0, h->sA>>>(h->top.U.p, h->n, h->row0, h->nloc, cols, buf_dev, rows_pad);
  BGP_LAUNCH_CHECK();
  BGP_CUDA(cudaStreamSynchronize(h->sA));
  return BGP_OK;
}

int bgp_hodlr_import_top(bgp_hodlr_t* h, const double* all_buf_dev, int64_t rows_pad) {
  if (!h) { set_error("null handle"); return BGP_ERR_INVALID; }
  BGP_TRY(require_top_pending(h, "import_top"));
  int64_t max_rows = 0;
  for (int64_t r : h->shard_rows) max_rows = std::max(max_rows, r);
  if (rows_pad < max_rows) {  // the slices would be read at the wrong offsets
    set_error("rows_pad %lld smaller than the largest shard (%lld rows)", (long long)rows_pad, (long long)max_rows);
    return BGP_ERR_INVALID;
  }
  const int64_t cols = top_cols(h);
  if (cols == 0) return BGP_OK;
  for (size_t s = 0; s < h->shard_rows.size(); ++s) {
    if ((int)s == h->opts.shard_rank) continue;  // own rows are already in place
    unpack_rows_kernel<<<1184, 256, 0, h->sA>>>(h->top.U.p, h->n, h->shard_row0[s], h->shard_rows[s], cols,
                                                all_buf_dev + (int64_t)s * cols * rows_pad, rows_pad);
    BGP_LAUNCH_CHECK();
  }
  BGP_CUDA(cudaStreamSynchronize(h->sA));
  return BGP_OK;
}

int bgp_hodlr_finish_top(bgp_hodlr_t* h) {
  if (!h) { set_error("null handle"); return BGP_ERR_INVALID; }
  BGP_TRY(require_top_pending(h, "finish_top"));
  h->top_pending = false;
  return hodlr_finish_top_impl(h, false);
}

int bgp_hodlr_solve_local_dev(bgp_hodlr_t* h, double* b_dev, int64_t nrhs, int64_t ldb) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  BGP_TRY(hodlr_solve_dev(h, b_dev, nrhs, ldb, h->sA, 1));
  BGP_CUDA(cudaStreamSynchronize(h->sA));
  return BGP_OK;
}
int bgp_hodlr_solve_top_dev(bgp_hodlr_t* h, double* b_dev, int64_t nrhs, int64_t ldb) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  BGP_TRY(hodlr_solve_dev(h, b_dev, nrhs, ldb, h->sA, 2));
  BGP_CUDA(cudaStreamSynchronize(h->sA));
  return BGP_OK;
}


// ---- the symmetric factor on a host-exchange shard (include/bgp.h) -------------------------------------------------
// sym_stage: 1 between bgp_hodlr_sym_factor_local and bgp_hodlr_sym_finish_top, -1 after a failed local build.
static int require_sym_local(const bgp_hodlr* h, const char* what) {
  if (!h) { set_error("null handle"); return BGP_ERR_INVALID; }
  if (h->sym_stage == 1) return BGP_OK;
  if (h->sym_current) {
    set_error("%s: the symmetric factor is complete (bgp_hodlr_sym_finish_top was already called, or it was built "
              "whole)", what);
    return BGP_ERR_INVALID;
  }
  if (h->sym_stage < 0) {
    set_error("%s: the local part of the symmetric factor failed to build (see bgp_hodlr_sym_factor_local's error)",
              what);
    return BGP_ERR_NOT_COMPUTED;
  }
  set_error("%s: the local part of the symmetric factor has not been built (bgp_hodlr_sym_factor_local)", what);
  return BGP_ERR_NOT_COMPUTED;
}

int bgp_hodlr_sym_factor_local(bgp_hodlr_t* h) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  BGP_TRY(require_device());
  h->sym_current = false;
  h->sym_stage = -1;
  BGP_TRY(sym_prepare_handle(h, false));
  BGP_TRY(sym_local_handle(h));
  h->sym_stage = 1;
  return BGP_OK;
}

int bgp_hodlr_sym_export_top(bgp_hodlr_t* h, double* buf_dev, int64_t rows_pad) {
  BGP_TRY(require_sym_local(h, "sym_export_top"));
  if (rows_pad < h->nloc) {
    set_error("rows_pad %lld smaller than this shard (%lld rows)", (long long)rows_pad, (long long)h->nloc);
    return BGP_ERR_INVALID;
  }
  int64_t cols = 0;
  double* ptop = sym_top_panel(h->sym, &cols);
  if (cols == 0 || h->nloc == 0) return BGP_OK;
  pack_rows_kernel<<<1184, 256, 0, h->sA>>>(ptop, h->n, h->row0, h->nloc, cols, buf_dev, rows_pad);
  BGP_LAUNCH_CHECK();
  BGP_CUDA(cudaStreamSynchronize(h->sA));
  return BGP_OK;
}

int bgp_hodlr_sym_import_top(bgp_hodlr_t* h, const double* all_buf_dev, int64_t rows_pad) {
  BGP_TRY(require_sym_local(h, "sym_import_top"));
  int64_t max_rows = 0;
  for (int64_t r : h->shard_rows) max_rows = std::max(max_rows, r);
  if (rows_pad < max_rows) {
    set_error("rows_pad %lld smaller than the largest shard (%lld rows)", (long long)rows_pad, (long long)max_rows);
    return BGP_ERR_INVALID;
  }
  int64_t cols = 0;
  double* ptop = sym_top_panel(h->sym, &cols);
  if (cols == 0) return BGP_OK;
  for (size_t s = 0; s < h->shard_rows.size(); ++s) {
    if ((int)s == h->opts.shard_rank) continue;  // own rows are already in place
    unpack_rows_kernel<<<1184, 256, 0, h->sA>>>(ptop, h->n, h->shard_row0[s], h->shard_rows[s], cols,
                                                all_buf_dev + (int64_t)s * cols * rows_pad, rows_pad);
    BGP_LAUNCH_CHECK();
  }
  BGP_CUDA(cudaStreamSynchronize(h->sA));
  return BGP_OK;
}

int bgp_hodlr_sym_finish_top(bgp_hodlr_t* h, double* partial_logdet) {
  BGP_TRY(require_sym_local(h, "sym_finish_top"));
  h->sym_stage = -1;
  double ld = 0.0;
  BGP_TRY(sym_build_top(h->sym, h->opts.shard_rank == 0, h->sA, &ld));
  h->sym_stage = 0;
  h->sym_log_det = ld;
  h->sym_current = true;
  if (partial_logdet) *partial_logdet = ld;
  return BGP_OK;
}

// part 1 (local) or 2 (top) of W z / W^T z in place on a device block; an unsharded handle builds the factor on first
// use (part 1 is all of it there, part 2 nothing), a sharded one needs bgp_hodlr_sym_finish_top (or, with a matching
// communicator, bgp_hodlr_sym_factor) first
static int sym_apply_part_dev(bgp_hodlr* h, double* z_dev, int64_t nrhs, int64_t ldz, int32_t transpose, int part) {
  if (!h || !h->computed) { set_error("the solver has not been computed"); return BGP_ERR_NOT_COMPUTED; }
  if (h->opts.shard_count == 1) {
    BGP_TRY(sym_require(h, "the symmetric factor"));
  } else if (!h->sym_current) {
    set_error("the symmetric factor of this shard is not complete (bgp_hodlr_sym_finish_top)");
    return BGP_ERR_NOT_COMPUTED;
  }
  if (nrhs <= 0) return BGP_OK;
  if (ldz < h->n) { set_error("dimension mismatch: ldz < n"); return BGP_ERR_DIM; }
  if (!z_dev) { set_error("sym_apply: z_dev is null"); return BGP_ERR_INVALID; }
  BGP_TRY(sym_apply_dev(h->sym, z_dev, ldz, nrhs, transpose ? 1 : 0, part, h->sA));
  BGP_CUDA(cudaStreamSynchronize(h->sA));
  return BGP_OK;
}

int bgp_hodlr_sym_apply_local_dev(bgp_hodlr_t* h, double* z_dev, int64_t nrhs, int64_t ldz, int32_t transpose) {
  return sym_apply_part_dev(h, z_dev, nrhs, ldz, transpose, 1);
}

int bgp_hodlr_sym_apply_top_dev(bgp_hodlr_t* h, double* z_dev, int64_t nrhs, int64_t ldz, int32_t transpose) {
  return sym_apply_part_dev(h, z_dev, nrhs, ldz, transpose, 2);
}

}  // extern "C"
