// TEST INFRASTRUCTURE — NOT PRODUCT CODE.
//
// CPU restatement (Eigen-free C++17) of the reference's HODLR solver, used as the parity oracle for the
// CUDA path and as the "port" CPU baseline in bench.py.  Only tests/, __graft_entry__.smoke() and
// bench.py's cpu_baseline / --impl reference legs may load liboracle.so.
//
// Follows, step by step:
//   src/george/include/george/hodlr.h:29-66    Node constructor: geometry, pre-order recursion, shared rng
//   src/george/include/george/hodlr.h:136-221  low_rank_approx: randomised-row / max-residual-column ACA
//   src/george/include/george/hodlr.h:75-103   compute: post-order factorisation + up-sweep over ancestors
//   src/george/include/george/hodlr.h:223-235  factorize (leaf: dense + LDLT; inner: 2r x 2r S + full-pivot LU)
//   src/george/include/george/hodlr.h:237-254  apply_inverse (leaf solve | Woodbury correction)
//   src/george/include/george/hodlr.h:107-114  solve
//   src/george/solvers/_hodlr.cpp:55-94        Solver::compute (mt19937::seed(seed), diag = yerr^2)
//
// Third-party arithmetic that is NOT under /root/reference (un-vendored submodule vendor/eigen, libeigen @
// db61b8d47825e55e348a66e77cb9e1f1cbae066b): Eigen::LDLT and Eigen::FullPivLU.  They are restated here from
// their published algorithms (diagonal-pivoted LDL^T; complete-pivoting LU with the rank threshold
// eps * diagonalSize used by solve()).  PARITY PIN: the reference _hodlr extension cannot be built here, so this
// restatement is pinned (tests/test_oracle_hodlr.py) against (a) the reference's own dense tests
// (tests/test_solvers.py:29-62: slogdet / solve / inverse of the explicitly built matrix, with kernel entries from the
// reference's compiled kernel_interface), (b) the docs' golden log-likelihood 133.946394912
// (docs/tutorials/scaling.rst:76,91) and (c) the std::mt19937 / uniform_int_distribution words of SURVEY.md App. B.
// The ACA pivot sequence itself is pinned by nothing but this restatement ("parity unpinned" at that granularity).
//
// RNG: the reference uses libstdc++'s std::mt19937 + std::uniform_int_distribution<int>; we use the very same
// library classes, so the stream is identical by construction (GCC 13).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <memory>
#include <random>
#include <vector>

#include "kernels_oracle.h"

namespace oracle {

// column-major dense matrix
struct Mat {
  int rows = 0, cols = 0;
  std::vector<double> a;
  Mat() {}
  Mat(int r, int c) : rows(r), cols(c), a((size_t)r * c, 0.0) {}
  double& operator()(int i, int j) { return a[(size_t)j * rows + i]; }
  double operator()(int i, int j) const { return a[(size_t)j * rows + i]; }
  double* col(int j) { return a.data() + (size_t)j * rows; }
  const double* col(int j) const { return a.data() + (size_t)j * rows; }
};

// ---- Eigen::LDLT restated: P A P^T = L D L^T with the largest remaining diagonal entry as pivot ----------
struct LDLT {
  int n = 0;
  Mat L;                    // unit lower, strictly-lower part used
  std::vector<double> D;
  std::vector<int> perm;    // transpositions
  void compute(const Mat& A) {
    n = A.rows; L = A; D.assign(n, 0.0); perm.assign(n, 0);
    for (int k = 0; k < n; ++k) {
      int p = k; double best = std::abs(L(k, k));
      for (int i = k + 1; i < n; ++i) if (std::abs(L(i, i)) > best) { best = std::abs(L(i, i)); p = i; }
      perm[k] = p;
      if (p != k) {  // symmetric swap on the lower triangle
        for (int j = 0; j < k; ++j) std::swap(L(k, j), L(p, j));
        for (int i = p + 1; i < n; ++i) std::swap(L(i, k), L(i, p));
        for (int i = k + 1; i < p; ++i) std::swap(L(i, k), L(p, i));
        std::swap(L(k, k), L(p, p));
      }
      // left-looking update of column k (what Eigen's unblocked ldlt_inplace does)
      if (k > 0) {
        std::vector<double> t(k);
        for (int j = 0; j < k; ++j) t[j] = L(k, j) * D[j];
        double s = 0.0;
        for (int j = 0; j < k; ++j) s += t[j] * L(k, j);
        L(k, k) -= s;
        for (int j = 0; j < k; ++j) {
          const double tj = t[j];
          const double* lj = L.col(j);
          double* lk = L.col(k);
          for (int i = k + 1; i < n; ++i) lk[i] -= lj[i] * tj;
        }
      }
      D[k] = L(k, k);
      if (std::abs(D[k]) > 0.0) { double inv = 1.0 / D[k]; double* lk = L.col(k); for (int i = k + 1; i < n; ++i) lk[i] *= inv; }
    }
  }
  // x (n x nrhs, leading dimension ldx) solved in place
  void solve(double* x, int nrhs, int ldx) const {
    const double tiny = std::numeric_limits<double>::min();
    for (int c = 0; c < nrhs; ++c) {
      double* b = x + (size_t)c * ldx;
      for (int k = 0; k < n; ++k) if (perm[k] != k) std::swap(b[k], b[perm[k]]);
      for (int j = 0; j < n; ++j) { const double bj = b[j]; const double* lj = L.col(j); for (int i = j + 1; i < n; ++i) b[i] -= lj[i] * bj; }
      for (int j = 0; j < n; ++j) b[j] = (std::abs(D[j]) > tiny) ? b[j] / D[j] : 0.0;   // Eigen: pseudo-inverse of D
      for (int j = n - 1; j >= 0; --j) { const double* lj = L.col(j); double s = 0.0; for (int i = j + 1; i < n; ++i) s += lj[i] * b[i]; b[j] -= s; }
      for (int k = n - 1; k >= 0; --k) if (perm[k] != k) std::swap(b[k], b[perm[k]]);
    }
  }
};

// ---- Eigen::FullPivLU restated: P A Q = L U with complete pivoting; solve() truncates at the numerical rank ----
struct FullPivLU {
  int n = 0;
  Mat lu;
  std::vector<int> rowt, colt;
  double maxpivot = 0.0;
  int nonzero = 0;
  void compute(const Mat& A) {
    n = A.rows; lu = A; rowt.assign(n, 0); colt.assign(n, 0); maxpivot = 0.0; nonzero = n;
    for (int k = 0; k < n; ++k) {
      int pr = k, pc = k; double best = -1.0;
      for (int j = k; j < n; ++j) for (int i = k; i < n; ++i) { double v = std::abs(lu(i, j)); if (v > best) { best = v; pr = i; pc = j; } }
      if (best == 0.0) { nonzero = k; for (int i = k; i < n; ++i) { rowt[i] = i; colt[i] = i; } break; }
      if (best > maxpivot) maxpivot = best;
      rowt[k] = pr; colt[k] = pc;
      if (pr != k) for (int j = 0; j < n; ++j) std::swap(lu(k, j), lu(pr, j));
      if (pc != k) for (int i = 0; i < n; ++i) std::swap(lu(i, k), lu(i, pc));
      const double inv = 1.0 / lu(k, k);
      for (int i = k + 1; i < n; ++i) lu(i, k) *= inv;
      for (int j = k + 1; j < n; ++j) { const double ukj = lu(k, j); for (int i = k + 1; i < n; ++i) lu(i, j) -= lu(i, k) * ukj; }
    }
  }
  int rank() const {
    const double thr = std::abs(maxpivot) * std::numeric_limits<double>::epsilon() * n;
    int r = 0;
    for (int i = 0; i < nonzero; ++i) r += (std::abs(lu(i, i)) > thr);
    return r;
  }
  void solve(double* x, int nrhs, int ldx) const {
    const int r = rank();
    std::vector<double> c(n);
    for (int col = 0; col < nrhs; ++col) {
      double* b = x + (size_t)col * ldx;
      for (int i = 0; i < n; ++i) c[i] = b[i];
      for (int k = 0; k < n; ++k) if (rowt[k] != k) std::swap(c[k], c[rowt[k]]);
      for (int j = 0; j < n; ++j) { const double cj = c[j]; for (int i = j + 1; i < n; ++i) c[i] -= lu(i, j) * cj; }
      for (int j = r - 1; j >= 0; --j) { c[j] /= lu(j, j); const double cj = c[j]; for (int i = 0; i < j; ++i) c[i] -= lu(i, j) * cj; }
      for (int i = r; i < n; ++i) c[i] = 0.0;
      for (int k = n - 1; k >= 0; --k) if (colt[k] != k) std::swap(c[k], c[colt[k]]);
      for (int i = 0; i < n; ++i) b[i] = c[i];
    }
  }
};

struct Solver;

struct Node {
  Solver* S;
  Node* parent;
  std::unique_ptr<Node> child[2];
  int start, size, direction, rank = 0, depth, id;
  bool is_leaf;
  Mat U[2], V[2];
  FullPivLU lu;
  LDLT ldlt;
  double log_det = 0.0;
  int rng_draws = 0, dense_fallback = 0;
  std::vector<int> piv_rows, piv_cols;
};

struct Solver {
  Program prog;
  int n = 0, ndim = 0, min_size = 100, rng_mode = BGP_RNG_REFERENCE;
  int exhaust_mode = BGP_EXHAUST_DENSE;  // BGP_EXHAUST_LOWRANK: the documented deviation of the CUDA path (DESIGN.md §2), restated
                                         // here so that the two can be compared one to one in that mode as well
  uint32_t seed = 42;
  double tol = 0.1;
  std::vector<double> x, diag;
  std::unique_ptr<Node> root;
  std::vector<Node*> preorder;
  double log_det = 0.0;
  uint64_t n_evals = 0;

  inline double K(int i, int j) {  // SolverMatrix::get_value, _hodlr.cpp:24-29
    ++n_evals;
    return program_value(prog, &x[(size_t)i * ndim], &x[(size_t)j * ndim]);
  }
};

// seed of the private stream of node `id` in BGP_RNG_PER_NODE mode (id = pre-order index; the root keeps `seed`).
static inline uint32_t node_seed(uint32_t seed, int id) { return seed + 0x9E3779B9u * (uint32_t)id; }

// hodlr.h:136-221
static int low_rank_approx(Solver* S, Node* nd, int start_row, int n_rows, int start_col, int n_cols, double tol,
                           std::mt19937& random, Mat& U_out, Mat& V_out) {
  const int max_rank = std::min(n_rows, n_cols);
  std::vector<std::vector<double>> U, V;  // columns, grown on demand (the reference pre-allocates n x max_rank)
  int rank = 0;
  double norm = 0.0;
  const double tol2 = tol * tol;
  std::vector<int> index(n_rows);
  for (int n = 0; n < n_rows; ++n) index[n] = n;
  std::vector<double> v(n_cols), u(n_rows);

  while (true) {
    int i, j = 0, k;
    do {
      if (index.empty()) {  // hodlr.h:161-176 dense fallback
        nd->dense_fallback = 1;
        if (S->exhaust_mode == BGP_EXHAUST_LOWRANK) {
          // NOT the reference: every row has been tried and none has a residual entry >= 1e-14, so the factors found
          // so far reproduce the block to 1e-14 per entry; keep them instead of storing the block densely.
          U_out = Mat(n_rows, rank); V_out = Mat(n_cols, rank);
          for (int q = 0; q < rank; ++q) { std::memcpy(U_out.col(q), U[q].data(), sizeof(double) * n_rows); std::memcpy(V_out.col(q), V[q].data(), sizeof(double) * n_cols); }
          return rank;
        }
        U_out = Mat(n_rows, max_rank); V_out = Mat(n_cols, max_rank);
        if (n_cols <= n_rows) {
          for (int m = 0; m < n_cols; ++m) { V_out(m, m) = 1.0; for (int n = 0; n < n_rows; ++n) U_out(n, m) = S->K(start_row + n, start_col + m); }
        } else {
          for (int n = 0; n < n_rows; ++n) { U_out(n, n) = 1.0; for (int m = 0; m < n_cols; ++m) V_out(m, n) = S->K(start_row + n, start_col + m); }
        }
        return max_rank;
      }
      std::uniform_int_distribution<int> uniform_dist(0, (int)index.size() - 1);
      k = uniform_dist(random);
      nd->rng_draws++;
      i = index[k];
      index[k] = index.back();
      index.pop_back();

      for (int n = 0; n < n_cols; ++n) v[n] = S->K(start_row + i, start_col + n);
      for (int q = 0; q < rank; ++q) { const double uiq = U[q][i]; const double* vq = V[q].data(); for (int n = 0; n < n_cols; ++n) v[n] -= uiq * vq[n]; }
      // first max, as Eigen's maxCoeff, with a NaN counted as +inf (NOT the reference, DESIGN.md §2: Eigen only lets a
      // NaN at column 0 win): the first NaN wins and an all-NaN row pivots on column 0 instead of a stale j
      double best = -1.0;
      for (int n = 0; n < n_cols; ++n) {
        const double a = std::isnan(v[n]) ? HUGE_VAL : std::abs(v[n]);
        if (a > best) { best = a; j = n; }
      }
    } while (std::abs(v[j]) < 1e-14);  // a NaN pivot is accepted

    const double pivot = v[j];
    for (int n = 0; n < n_cols; ++n) v[n] /= pivot;
    for (int n = 0; n < n_rows; ++n) u[n] = S->K(start_row + n, start_col + j);
    for (int q = 0; q < rank; ++q) { const double vjq = V[q][j]; const double* uq = U[q].data(); for (int n = 0; n < n_rows; ++n) u[n] -= vjq * uq[n]; }
    U.push_back(u); V.push_back(v);
    nd->piv_rows.push_back(i); nd->piv_cols.push_back(j);
    rank++;
    if (rank >= max_rank) break;

    double un = 0.0, vn = 0.0;
    for (int n = 0; n < n_rows; ++n) un += u[n] * u[n];
    for (int n = 0; n < n_cols; ++n) vn += v[n] * v[n];
    const double rowcol_norm = un * vn;
    if (rowcol_norm < tol2 * norm) break;
    norm += rowcol_norm;
    if (rank > 1) {
      double mu = 0.0, mv = 0.0;
      for (int q = 0; q < rank - 1; ++q) {
        double s = 0.0; const double* uq = U[q].data();
        for (int n = 0; n < n_rows; ++n) s += uq[n] * u[n];
        mu = std::max(mu, std::abs(s));
        s = 0.0; const double* vq = V[q].data();
        for (int n = 0; n < n_cols; ++n) s += vq[n] * v[n];
        mv = std::max(mv, std::abs(s));
      }
      norm += 2.0 * mu + 2.0 * mv;
    }
  }
  U_out = Mat(n_rows, rank); V_out = Mat(n_cols, rank);
  for (int q = 0; q < rank; ++q) { std::memcpy(U_out.col(q), U[q].data(), sizeof(double) * n_rows); std::memcpy(V_out.col(q), V[q].data(), sizeof(double) * n_cols); }
  return rank;
}

// hodlr.h:29-66
static std::unique_ptr<Node> build(Solver* S, int start, int size, std::mt19937& random, int direction, Node* parent, int depth) {
  std::unique_ptr<Node> nd(new Node());
  nd->S = S; nd->parent = parent; nd->start = start; nd->size = size; nd->direction = direction; nd->depth = depth;
  nd->id = (int)S->preorder.size();
  S->preorder.push_back(nd.get());
  const int half = size / 2;
  if (half >= S->min_size) {
    nd->is_leaf = false;
    if (S->rng_mode == BGP_RNG_PER_NODE) {
      std::mt19937 own; own.seed(node_seed(S->seed, nd->id));
      nd->rank = low_rank_approx(S, nd.get(), start + half, size - half, start, half, S->tol, own, nd->U[1], nd->V[0]);
    } else {
      nd->rank = low_rank_approx(S, nd.get(), start + half, size - half, start, half, S->tol, random, nd->U[1], nd->V[0]);
    }
    nd->U[0] = nd->V[0];
    nd->V[1] = nd->U[1];
    nd->child[0] = build(S, start, half, random, 0, nd.get(), depth + 1);
    nd->child[1] = build(S, start + half, size - half, random, 1, nd.get(), depth + 1);
  } else {
    nd->is_leaf = true;
  }
  return nd;
}

// hodlr.h:237-254.  x: rows [row0, row0+rows) of some matrix, column-major, leading dimension ldx; `start` is the
// global index of x's first row.
static void apply_inverse(const Node* nd, double* x, int nrhs, int ldx, int start) {
  const int off = nd->start - start;
  if (nd->is_leaf) { nd->ldlt.solve(x + off, nrhs, ldx); return; }
  const int s1 = nd->size / 2, s2 = nd->size - s1, r = nd->rank;
  if (r == 0) return;
  Mat temp(2 * r, nrhs);
  for (int c = 0; c < nrhs; ++c) {
    const double* x1 = x + (size_t)c * ldx + off;
    const double* x2 = x1 + s1;
    for (int q = 0; q < r; ++q) {
      const double* v1 = nd->V[1].col(q); double s = 0.0;
      for (int i = 0; i < s2; ++i) s += v1[i] * x2[i];
      temp(q, c) = s;
      const double* v0 = nd->V[0].col(q); s = 0.0;
      for (int i = 0; i < s1; ++i) s += v0[i] * x1[i];
      temp(r + q, c) = s;
    }
  }
  nd->lu.solve(temp.a.data(), nrhs, 2 * r);
  for (int c = 0; c < nrhs; ++c) {
    double* x1 = x + (size_t)c * ldx + off;
    double* x2 = x1 + s1;
    for (int q = 0; q < r; ++q) {
      const double t0 = temp(q, c), t1 = temp(r + q, c);
      const double* u0 = nd->U[0].col(q); for (int i = 0; i < s1; ++i) x1[i] -= u0[i] * t0;
      const double* u1 = nd->U[1].col(q); for (int i = 0; i < s2; ++i) x2[i] -= u1[i] * t1;
    }
  }
}

// hodlr.h:223-235 + 75-103
static void compute(Node* nd) {
  Solver* S = nd->S;
  nd->log_det = 0.0;
  if (!nd->is_leaf) {
    compute(nd->child[0].get());
    compute(nd->child[1].get());
    nd->log_det = nd->child[0]->log_det + nd->child[1]->log_det;
  }
  if (nd->is_leaf) {
    Mat A(nd->size, nd->size);  // get_exact_matrix, hodlr.h:122-133
    for (int n = 0; n < nd->size; ++n) {
      A(n, n) = S->diag[nd->start + n] + S->K(nd->start + n, nd->start + n);
      for (int m = n + 1; m < nd->size; ++m) { double v = S->K(nd->start + m, nd->start + n); A(m, n) = v; A(n, m) = v; }
    }
    nd->ldlt.compute(A);
    for (int n = 0; n < nd->size; ++n) nd->log_det += std::log(std::abs(nd->ldlt.D[n]));
  } else {
    const int r = nd->rank, s1 = nd->size / 2, s2 = nd->size - s1;
    Mat Sm(2 * r, 2 * r);
    for (int i = 0; i < 2 * r; ++i) Sm(i, i) = 1.0;
    for (int a = 0; a < r; ++a) for (int b = 0; b < r; ++b) {
      double s = 0.0; const double* va = nd->V[1].col(a); const double* ub = nd->U[1].col(b);
      for (int i = 0; i < s2; ++i) s += va[i] * ub[i];
      Sm(a, r + b) = s;
      s = 0.0; va = nd->V[0].col(a); ub = nd->U[0].col(b);
      for (int i = 0; i < s1; ++i) s += va[i] * ub[i];
      Sm(r + a, b) = s;
    }
    nd->lu.compute(Sm);
    for (int n = 0; n < 2 * r; ++n) nd->log_det += std::log(std::abs(nd->lu.lu(n, n)));
  }
  Node* node = nd->parent;
  int start = nd->start, ind = nd->direction;
  const Node* me = nd;
  while (node) {
    Mat& Ua = node->U[ind];
    // rows of Ua cover [node->start + (ind ? half : 0), ...); `start` below is the global index of Ua's first row
    const int ua_start = node->start + (ind ? node->size / 2 : 0);
    if (Ua.cols > 0) apply_inverse(me, Ua.a.data(), Ua.cols, Ua.rows, ua_start);
    (void)start;
    ind = node->direction;
    node = node->parent;
  }
}

// hodlr.h:107-114
static void solve(const Node* nd, double* x, int nrhs, int ldx) {
  if (!nd->is_leaf) { solve(nd->child[0].get(), x, nrhs, ldx); solve(nd->child[1].get(), x, nrhs, ldx); }
  apply_inverse(nd, x, nrhs, ldx, 0);
}

}  // namespace oracle

using namespace oracle;

extern "C" {

int oracle_num_params(const bgp_kernel_spec_t* spec) {
  Program P; if (build_program(spec, &P)) return -1; return P.n_params_total;
}

// kernel_interface.cpp:47-60
int oracle_value_general(const bgp_kernel_spec_t* spec, const double* x1, int64_t n1, const double* x2, int64_t n2, double* out) {
  Program P; if (build_program(spec, &P)) return 1;
  const int d = P.ndim;
  for (int64_t i = 0; i < n1; ++i) for (int64_t j = 0; j < n2; ++j) out[i * n2 + j] = program_value(P, x1 + i * d, x2 + j * d);
  return 0;
}
// kernel_interface.cpp:62-77
int oracle_value_symmetric(const bgp_kernel_spec_t* spec, const double* x, int64_t n, double* out) {
  Program P; if (build_program(spec, &P)) return 1;
  const int d = P.ndim;
  for (int64_t i = 0; i < n; ++i) {
    out[i * n + i] = program_value(P, x + i * d, x + i * d);
    for (int64_t j = i + 1; j < n; ++j) { double v = program_value(P, x + i * d, x + j * d); out[i * n + j] = v; out[j * n + i] = v; }
  }
  return 0;
}
// kernel_interface.cpp:79-90
int oracle_value_diagonal(const bgp_kernel_spec_t* spec, const double* x1, const double* x2, int64_t n, double* out) {
  Program P; if (build_program(spec, &P)) return 1;
  const int d = P.ndim;
  for (int64_t i = 0; i < n; ++i) out[i] = program_value(P, x1 + i * d, x2 + i * d);
  return 0;
}
// kernel_interface.cpp:92-107
int oracle_gradient_general(const bgp_kernel_spec_t* spec, const uint32_t* which, const double* x1, int64_t n1,
                            const double* x2, int64_t n2, double* out) {
  Program P; if (build_program(spec, &P)) return 1;
  const int d = P.ndim, np = P.n_params_total;
  for (int64_t i = 0; i < n1; ++i) for (int64_t j = 0; j < n2; ++j)
    program_gradient(P, x1 + i * d, x2 + j * d, which, out + (i * n2 + j) * np);
  return 0;
}

// kernel_interface.cpp:127-157; side = 1 -> x1_gradient_general, side = 2 -> x2_gradient_general; out (n1, n2, ndim)
int oracle_x_gradient_general(const bgp_kernel_spec_t* spec, int side, const double* x1, int64_t n1, const double* x2,
                              int64_t n2, double* out) {
  Program P; if (build_program(spec, &P)) return 1;
  const int d = P.ndim;
  for (int64_t i = 0; i < n1; ++i) for (int64_t j = 0; j < n2; ++j)
    program_x_gradient(P, side, x1 + i * d, x2 + j * d, out + (i * n2 + j) * d);
  return 0;
}

// _hodlr.cpp:55-94
void* oracle_hodlr_compute2(const bgp_kernel_spec_t* spec, const double* x, int64_t n, int32_t ndim, const double* yerr,
                            int32_t min_size, double tol, int32_t seed, int32_t rng_mode, int32_t exhaust_mode) {
  Solver* S = new Solver();
  if (build_program(spec, &S->prog) || S->prog.ndim != ndim) { delete S; return nullptr; }
  S->n = (int)n; S->ndim = ndim; S->min_size = min_size; S->tol = tol; S->seed = (uint32_t)seed; S->rng_mode = rng_mode;
  S->exhaust_mode = exhaust_mode;
  S->x.assign(x, x + (size_t)n * ndim);
  S->diag.resize(n);
  for (int64_t i = 0; i < n; ++i) S->diag[i] = yerr[i] * yerr[i];
  std::mt19937 random;
  random.seed((uint32_t)seed);
  S->root = build(S, 0, (int)n, random, 0, nullptr, 0);
  compute(S->root.get());
  S->log_det = S->root->log_det;
  return S;
}
void* oracle_hodlr_compute(const bgp_kernel_spec_t* spec, const double* x, int64_t n, int32_t ndim, const double* yerr,
                           int32_t min_size, double tol, int32_t seed, int32_t rng_mode) {
  return oracle_hodlr_compute2(spec, x, n, ndim, yerr, min_size, tol, seed, rng_mode, BGP_EXHAUST_DENSE);
}
void oracle_hodlr_free(void* h) { delete (Solver*)h; }
double oracle_hodlr_log_determinant(void* h) { return ((Solver*)h)->log_det; }
uint64_t oracle_hodlr_num_evals(void* h) { return ((Solver*)h)->n_evals; }
// b: (n, nrhs) column-major, solved in place (_hodlr.cpp:156-164)
void oracle_hodlr_apply_inverse(void* h, double* b, int64_t nrhs, int64_t ldb) {
  Solver* S = (Solver*)h;
  solve(S->root.get(), b, (int)nrhs, (int)ldb);
}
double oracle_hodlr_dot_solve(void* h, const double* y) {  // _hodlr.cpp:178-182
  Solver* S = (Solver*)h;
  std::vector<double> a(y, y + S->n);
  solve(S->root.get(), a.data(), 1, S->n);
  double s = 0.0;
  for (int i = 0; i < S->n; ++i) s += y[i] * a[i];
  return s;
}
int64_t oracle_hodlr_num_nodes(void* h) { return (int64_t)((Solver*)h)->preorder.size(); }
void oracle_hodlr_node_info(void* h, bgp_hodlr_node_info_t* out) {
  Solver* S = (Solver*)h;
  for (size_t i = 0; i < S->preorder.size(); ++i) {
    const Node* nd = S->preorder[i];
    out[i].start = nd->start; out[i].size = nd->size; out[i].half = nd->size / 2; out[i].is_leaf = nd->is_leaf;
    out[i].parent = nd->parent ? nd->parent->id : -1; out[i].direction = nd->direction; out[i].depth = nd->depth;
    out[i].rank = nd->rank; out[i].rng_draws = nd->rng_draws; out[i].dense_fallback = nd->dense_fallback;
  }
}
int oracle_hodlr_node_pivots(void* h, int64_t node, int32_t* rows, int32_t* cols) {
  Solver* S = (Solver*)h;
  if (node < 0 || node >= (int64_t)S->preorder.size()) return 1;
  const Node* nd = S->preorder[node];
  for (size_t k = 0; k < nd->piv_rows.size(); ++k) { rows[k] = nd->piv_rows[k]; cols[k] = nd->piv_cols[k]; }
  return (int)nd->piv_rows.size();
}

// libstdc++ stream probes (SURVEY.md App. B golden words)
void oracle_mt19937_words(uint32_t seed, int n, uint32_t* out) { std::mt19937 r; r.seed(seed); for (int i = 0; i < n; ++i) out[i] = (uint32_t)r(); }
void oracle_uniform_ints(uint32_t seed, int n, const int32_t* sizes, int32_t* out) {
  std::mt19937 r; r.seed(seed);
  for (int i = 0; i < n; ++i) { std::uniform_int_distribution<int> d(0, sizes[i] - 1); out[i] = d(r); }
}

}  // extern "C"
