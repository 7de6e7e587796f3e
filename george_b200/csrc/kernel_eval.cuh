// kernel_eval.cuh — device-side covariance evaluation from the POD kernel program.
//
// The reference evaluates k(x1, x2) through a heap tree of virtual C++ objects
// (src/george/include/george/kernels.h:21-40, Sum :75-109, Product :111-163, per-kernel classes below that; metrics in
// metrics.h:71-253).  Here the tree is a postfix program that a thread interprets with a small register stack;
// re-parametrisations (exp(-log M), pi * exp(-log P), ...) are done ONCE on the host with the same libm calls the
// reference makes (update_reparams(), Metric::set_parameter metrics.h:46-49), so the device only sees the digested
// constants and differs from the CPU path by the <=2 ulp of CUDA's exp/sin/cos/pow.
#pragma once

#include <cfloat>

#include "common.cuh"
#include "user_kernels.cuh"  // generated from kernels/*.yml (tools/generate_kernels.py)

namespace bgp {

#define BGP_MAX_LEAVES 16
#define BGP_STACK 8  // operand-stack depth of the interpreter (validated on the host)

struct DevLeaf {
  int kernel_type, metric_type, naxes, blocked, n_params, n_metric, param_off, _pad;
  int axes[BGP_MAX_DIM];
  double p[4];                  // raw parameters
  double rp[2];                 // re-parametrised constants
  double mvec[BGP_MAX_METRIC];  // metric vector_ (metrics.h:46-49,170-180)
  double mn[BGP_MAX_DIM], mx[BGP_MAX_DIM];
};

struct DevProgram {
  int n_nodes, ndim, n_params_total, n_leaves;
  int flags;  // bit0: 1-D input and every leaf depends on d = x1 - x2 only (fast path)
  int shape;  // 0 generic; otherwise BGP_SHAPE_*: the whole program is  sc * f(d*d*sm)  with f a stationary profile,
              // or one of the two-term 1-D forms  sc*f(d*d*sm) + sc2*ExpSine2  /  (sc*f(d*d*sm)) * ExpSine2
  int _pad[2];
  double sc, sm;
  double sc2, sg, sw;  // two-term shapes: scale of the periodic term, its Gamma and pi / period (kernels.h:1513-1537)
  signed char code[BGP_MAX_NODES];  // >=0: leaf index, -1: sum, -2: product
  DevLeaf leaf[BGP_MAX_LEAVES];
};

// number of bytes of a program that are live (header + used leaves): what kernels stage into shared memory
__host__ __device__ inline size_t program_bytes(int n_leaves) {
  return offsetof(DevProgram, leaf) + sizeof(DevLeaf) * (size_t)n_leaves;
}

// host: digest + validate a bgp_kernel_spec_t (replaces parser.h:14-509 + update_reparams())
int build_dev_program(const bgp_kernel_spec_t* spec, DevProgram* out);

// The tile kernels (the kernel-matrix builds of kmat.cu, the matvec of kmat_ops.cu) stage a tile's coordinates in
// dynamic shared memory next to the program, a block that grows with ndim.  Each comes in two instantiations: `staged`
// (footprint staged_bytes) and one that reads the coordinates from global memory (unstaged_bytes), with the same
// evaluation order and results.  The staged one runs whenever it fits under the kernel's cap, so no input dimension is
// too wide for these paths.  Returns the instantiation to launch, with its attribute set and *smem its footprint.
template <class Kernel>
Kernel tile_kernel_for(Kernel staged, Kernel unstaged, size_t staged_bytes, size_t unstaged_bytes, size_t cap,
                       size_t* smem) {
  const bool fits = staged_bytes <= cap;
  *smem = fits ? staged_bytes : unstaged_bytes;
  const Kernel k = fits ? staged : unstaged;
  // (the attribute is per device / context: set it on every call, it is cheap)
  cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)*smem);
  return k;
}

#ifdef __CUDACC__

// cooperative copy of the live part of the program into shared memory (all threads of the CTA must call)
__device__ __forceinline__ void stage_program(DevProgram* dst_smem, const DevProgram* __restrict__ src) {
  const int nl = src->n_leaves;
  const int words = (int)(program_bytes(nl) / 4);
  const uint32_t* s = reinterpret_cast<const uint32_t*>(src);
  uint32_t* d = reinterpret_cast<uint32_t*>(dst_smem);
  for (int i = threadIdx.x; i < words; i += blockDim.x) d[i] = s[i];
}

__device__ __forceinline__ bool general_is_diag(int i) {
  for (int j = 0, d = 2; j <= i; j += d, ++d)
    if (i == j) return true;
  return false;
}

// r2 = (x1-x2)^T M^-1 (x1-x2) on the leaf's axes.  metrics.h:76-85 | 108-117 | 182-197
__device__ __forceinline__ double metric_r2(const DevLeaf& L, const double* x1, const double* x2) {
  double r2 = 0.0;
  if (L.metric_type == BGP_METRIC_ISOTROPIC) {
    for (int i = 0; i < L.naxes; ++i) {
      const double d = x1[L.axes[i]] - x2[L.axes[i]];
      r2 += d * d;
    }
    return r2 * L.mvec[0];
  }
  if (L.metric_type == BGP_METRIC_AXIS_ALIGNED) {
    for (int i = 0; i < L.naxes; ++i) {
      const double d = x1[L.axes[i]] - x2[L.axes[i]];
      r2 += d * d * L.mvec[i];
    }
    return r2;
  }
  // general: forward substitution with the packed inverse-diagonal Cholesky factor (metrics.h:144-151)
  double r[BGP_MAX_DIM];
  const int n = L.naxes;
  int k = 0;
  for (int i = 0; i < n; ++i) {
    double b = x1[L.axes[i]] - x2[L.axes[i]];
    for (int j = 0; j < i; ++j, ++k) b -= L.mvec[k] * r[j];
    b *= L.mvec[k++];
    r[i] = b;
    r2 += b * b;
  }
  return r2;
}

// metric value + gradient wrt the metric parameters.  metrics.h:87-91 | 119-131 | 201-231
__device__ inline double metric_r2_grad(const DevLeaf& L, const double* x1, const double* x2, double* grad) {
  double r2 = 0.0;
  if (L.metric_type == BGP_METRIC_ISOTROPIC) {
    r2 = metric_r2(L, x1, x2);
    grad[0] = -r2;
    return r2;
  }
  if (L.metric_type == BGP_METRIC_AXIS_ALIGNED) {
    for (int i = 0; i < L.naxes; ++i) {
      double d = x1[L.axes[i]] - x2[L.axes[i]];
      d = d * d * L.mvec[i];
      r2 += d;
      grad[i] = -d;
    }
    return r2;
  }
  double r[BGP_MAX_DIM], Lir[BGP_MAX_DIM];
  const int n = L.naxes;
  int k = 0;
  for (int i = 0; i < n; ++i) {
    double b = x1[L.axes[i]] - x2[L.axes[i]];
    for (int j = 0; j < i; ++j, ++k) b -= L.mvec[k] * r[j];
    b *= L.mvec[k++];
    r[i] = b;
    Lir[i] = b;
    r2 += b * b;
  }
  // backward substitution (metrics.h:153-164)
  const int k0 = (n + 1) * n / 2;
  for (int i = n - 1; i >= 0; --i) {
    int kk = k0 - n + i;
    for (int j = n - 1; j > i; --j) {
      r[i] -= L.mvec[kk] * r[j];
      kk -= j;
    }
    r[i] *= L.mvec[kk];
  }
  k = 0;
  for (int i = 0; i < n; ++i) {
    grad[k] = -2 * r[i] * Lir[i] * exp(L.mvec[k]);  // metrics.h:222 (sic: exp of the stored inverse-diagonal entry)
    k++;
    for (int j = i + 1; j < n; ++j) grad[k++] = -2 * r[j] * Lir[i];
  }
  return r2;
}

__device__ __forceinline__ bool out_of_block(const DevLeaf& L, const double* x1, const double* x2) {
  for (int i = 0; i < L.naxes; ++i) {
    const int j = L.axes[i];
    if (x1[j] < L.mn[i] || x1[j] > L.mx[i] || x2[j] < L.mn[i] || x2[j] > L.mx[i]) return true;
  }
  return false;
}

// radial profiles k(r2): kernels.h:1890-1894 ExpSquared | 2084-2090 Matern32 | 1319-1325 Matern52 | 651-655 Exp |
// 418-425 RationalQuadratic
__device__ __forceinline__ double radial_value(const DevLeaf& L, double r2) {
  switch (L.kernel_type) {
    case BGP_K_EXP_SQUARED: return exp(-0.5 * r2);
    case BGP_K_MATERN32: { const double r = sqrt(3.0 * r2); return (1.0 + r) * exp(-r); }
    case BGP_K_MATERN52: { const double r = sqrt(5.0 * r2); return (1 + r + 5.0 * r2 / 3.0) * exp(-r); }
    case BGP_K_EXP: return exp(-sqrt(r2));
    case BGP_K_RATIONAL_QUADRATIC: return pow(1 + 0.5 * r2 / L.rp[0], -L.rp[0]);
  }
  if (L.kernel_type >= BGP_K_USER0) return user::radial_value(L.kernel_type - BGP_K_USER0, r2, L.p, L.rp);
  return 0.0;
}
// dk/dr2: kernels.h:1912-1916 | 2108-2114 | 1343-1349 | Exp.yml | 454-461
__device__ __forceinline__ double radial_gradient(const DevLeaf& L, double r2) {
  switch (L.kernel_type) {
    case BGP_K_EXP_SQUARED: return -0.5 * exp(-0.5 * r2);
    case BGP_K_MATERN32: { const double r = sqrt(3.0 * r2); return -3.0 * 0.5 * exp(-r); }
    case BGP_K_MATERN52: { const double r = sqrt(5.0 * r2); return -5 * (1 + r) * exp(-r) / 6.0; }
    case BGP_K_EXP: { if (r2 < 2.220446049250313e-16) return 0.0; const double r = sqrt(r2); return -0.5 * exp(-r) / r; }
    case BGP_K_RATIONAL_QUADRATIC: return -0.5 * pow(1 + 0.5 * r2 / L.rp[0], -L.rp[0] - 1);
  }
  if (L.kernel_type >= BGP_K_USER0) return user::radial_gradient(L.kernel_type - BGP_K_USER0, r2, L.p, L.rp);
  return 0.0;
}

// per-axis value of the non-stationary kernels (summed over the leaf's axes, e.g. kernels.h:1720-1732)
__device__ __forceinline__ double axis_value(const DevLeaf& L, double x1, double x2) {
  switch (L.kernel_type) {
    case BGP_K_LINEAR: if (L.p[1] == 0.0) return L.rp[0]; return pow(x1 * x2, L.p[1]) * L.rp[0];
    case BGP_K_LOCAL_GAUSSIAN: { const double d1 = x1 - L.p[0], d2 = x2 - L.p[0]; return exp(-(d1 * d1 + d2 * d2) * L.rp[0]); }
    case BGP_K_EMPTY: return 0.0;
    case BGP_K_COSINE: return cos((x1 - x2) * L.rp[0]);
    case BGP_K_EXP_SINE2: { const double s = sin((x1 - x2) * L.rp[0]); return exp(-L.p[0] * s * s); }
    case BGP_K_CONSTANT: return L.rp[0];
    case BGP_K_POLYNOMIAL: if (L.p[1] == 0.0) return 1.0; return pow(x1 * x2 + L.rp[0], L.p[1]);
    case BGP_K_DOT_PRODUCT: return x1 * x2;
  }
  if (L.kernel_type >= BGP_K_USER0) return user::axis_value(L.kernel_type - BGP_K_USER0, x1, x2, L.p, L.rp);
  return 0.0;
}
__device__ inline double axis_param_gradient(const DevLeaf& L, int q, double x1, double x2) {
  switch (L.kernel_type) {
    case BGP_K_LINEAR: if (L.p[1] == 0.0) return -L.rp[0]; return -pow(x1 * x2, L.p[1]) * L.rp[0];
    case BGP_K_LOCAL_GAUSSIAN: {
      const double d1 = x1 - L.p[0], d2 = x2 - L.p[0];
      if (q == 0) return 2 * exp(-(d1 * d1 + d2 * d2) * L.rp[0]) * L.rp[0] * (d1 + d2);
      const double arg = (d1 * d1 + d2 * d2) * L.rp[0];
      return exp(-arg) * arg;
    }
    case BGP_K_COSINE: { const double r = L.rp[0] * (x1 - x2); return r * sin(r); }
    case BGP_K_EXP_SINE2: {
      if (q == 0) { const double s = sin((x1 - x2) * L.rp[0]), s2 = s * s; return -s2 * exp(-L.p[0] * s2); }
      const double arg = (x1 - x2) * L.rp[0], s = sin(arg), c = cos(arg), A = exp(-L.p[0] * s * s);
      return 2 * L.p[0] * arg * c * s * A;
    }
    case BGP_K_CONSTANT: return L.rp[0];
    case BGP_K_POLYNOMIAL: if (L.p[1] == 0.0) return 0.0; return L.rp[0] * pow(x1 * x2 + L.rp[0], L.p[1] - 1.0) * L.p[1];
  }
  if (L.kernel_type >= BGP_K_USER0) return user::axis_param_gradient(L.kernel_type - BGP_K_USER0, q, x1, x2, L.p, L.rp);
  return 0.0;
}

__device__ __forceinline__ double leaf_value(const DevLeaf& L, const double* x1, const double* x2) {
  if (L.metric_type != BGP_METRIC_NONE) {
    if (L.blocked && out_of_block(L, x1, x2)) return 0.0;
    return radial_value(L, metric_r2(L, x1, x2));
  }
  double v = 0.0;
  for (int i = 0; i < L.naxes; ++i) v += axis_value(L, x1[L.axes[i]], x2[L.axes[i]]);
  return v;
}

// Fast path for 1-D inputs whose leaves all depend on d = x1 - x2 only (stationary kernels with a scalar metric,
// ExpSine2, Cosine, Constant): no axis indirection, no metric loops.  Same arithmetic, same order, as the general path.
#define BGP_FLAG_FAST1D 1
enum {
  BGP_SHAPE_GENERIC = 0, BGP_SHAPE_EXPSQ = 1, BGP_SHAPE_M32 = 2, BGP_SHAPE_M52 = 3, BGP_SHAPE_EXP = 4,
  // two-term programs on 1-D inputs (the usual quasi-periodic models):  c*A + c2*ExpSine2  and  (c*A) * ExpSine2
  BGP_SHAPE_SUM_EXPSQ_ES2 = 5, BGP_SHAPE_SUM_M32_ES2 = 6, BGP_SHAPE_PROD_EXPSQ_ES2 = 7, BGP_SHAPE_PROD_M32_ES2 = 8,
  BGP_NUM_SHAPES = 9
};
__host__ __device__ constexpr int shape_profile(int shape) {  // the stationary profile a shape is built on
  return shape <= BGP_SHAPE_EXP ? shape
         : (shape == BGP_SHAPE_SUM_EXPSQ_ES2 || shape == BGP_SHAPE_PROD_EXPSQ_ES2) ? (int)BGP_SHAPE_EXPSQ : (int)BGP_SHAPE_M32;
}
__host__ __device__ constexpr bool shape_is_sum(int shape) { return shape == BGP_SHAPE_SUM_EXPSQ_ES2 || shape == BGP_SHAPE_SUM_M32_ES2; }
__host__ __device__ constexpr bool shape_is_prod(int shape) { return shape == BGP_SHAPE_PROD_EXPSQ_ES2 || shape == BGP_SHAPE_PROD_M32_ES2; }
// |k| has a usable decreasing bound in the distance (everything but the sums with a periodic term, which never decay)
__host__ __device__ constexpr bool shape_has_bound(int shape) { return shape != BGP_SHAPE_GENERIC && !shape_is_sum(shape); }

// radial profile f(r2) of the specialised evaluators.  exp(-t) rounds to exactly 0 in double for t > 745.14: far-apart
// pairs (the bulk of every large off-diagonal block) skip the software exp/sqrt; the branch is warp-uniform because a
// warp sweeps 32 neighbouring points.  Same expressions, same order, as leaf_value_1d / radial_value.  At r2 = +inf
// the Matern forms are (1 + inf) * exp(-inf) = NaN there, so their cutoffs stop at DBL_MAX; EXPSQ and EXP give 0.
template <int PROFILE>
__device__ __forceinline__ double profile_value(double r2) {
  if (PROFILE == BGP_SHAPE_EXPSQ) return (r2 > 1490.4) ? 0.0 : exp(-0.5 * r2);
  if (PROFILE == BGP_SHAPE_M32) {
    if (r2 > 185200.0 && r2 <= DBL_MAX) return 0.0;  // sqrt(3 r2) > 745.3
    const double r = sqrt(3.0 * r2);
    return (1.0 + r) * exp(-r);
  }
  if (PROFILE == BGP_SHAPE_M52) {
    if (r2 > 111100.0 && r2 <= DBL_MAX) return 0.0;  // sqrt(5 r2) > 745.3
    const double r = sqrt(5.0 * r2);
    return (1 + r + 5.0 * r2 / 3.0) * exp(-r);
  }
  return (r2 > 555400.0) ? 0.0 : exp(-sqrt(r2));  // sqrt(r2) > 745.2
}

// compile-time specialised evaluators for the commonest programs on 1-D inputs: the interpreter disappears and
// independent evaluations can be interleaved by the compiler.  The operators of the two-term shapes are spelled with
// round-to-nearest intrinsics so that no multiply-add contraction can make them differ from the interpreter, which
// applies Sum / Product (kernels.h:78-80, 114-116) one node at a time.
template <int SHAPE>
struct ScaledProfile1D {
  double c, m, c2, g, w;
  __device__ __forceinline__ explicit ScaledProfile1D(const DevProgram& P) : c(P.sc), m(P.sm), c2(P.sc2), g(P.sg), w(P.sw) {}
  __device__ __forceinline__ ScaledProfile1D(double c_, double m_) : c(c_), m(m_), c2(0.0), g(0.0), w(0.0) {}
  __device__ __forceinline__ double operator()(const double* x1, const double* x2) const {
    const double d = x1[0] - x2[0];
    const double r2 = d * d * m;
    const double a = __dmul_rn(c, profile_value<shape_profile(SHAPE)>(r2));
    if (SHAPE <= BGP_SHAPE_EXP) return a;
    const double s = sin(d * w);
    const double e = exp(-g * s * s);
    if (shape_is_sum(SHAPE)) return __dadd_rn(a, __dmul_rn(c2, e));
    return __dmul_rn(a, e);
  }
  // upper bound of |k(x1, x2)| over all pairs at a distance in [gap, far] (monotone profiles; the periodic factor is
  // <= 1).  NaN, which keeps every candidate, when some such pair may evaluate to NaN: far not finite (a non-finite
  // coordinate), or r2 / the periodic phase overflowing to inf at distance far.  Only meaningful when shape_has_bound(SHAPE).
  __device__ __forceinline__ double bound(double gap, double far) const {
    if (!(far * far * m <= DBL_MAX) || (shape_is_prod(SHAPE) && !(fabs(far * w) <= DBL_MAX)))
      return __longlong_as_double(0x7ff8000000000000ll);
    double b = fabs(c) * profile_value<shape_profile(SHAPE)>(gap * gap * m);
    if (shape_is_prod(SHAPE) && g < 0.0) b *= exp(-g);  // exp(-Gamma sin^2) <= 1 only for Gamma >= 0
    return b;
  }
};
__device__ __forceinline__ double leaf_value_1d(const DevLeaf& L, double d) {
  switch (L.kernel_type) {
    case BGP_K_EXP_SQUARED: { const double r2 = d * d * L.mvec[0]; return exp(-0.5 * r2); }
    case BGP_K_MATERN32: { const double r2 = d * d * L.mvec[0]; const double r = sqrt(3.0 * r2); return (1.0 + r) * exp(-r); }
    case BGP_K_MATERN52: { const double r2 = d * d * L.mvec[0]; const double r = sqrt(5.0 * r2); return (1 + r + 5.0 * r2 / 3.0) * exp(-r); }
    case BGP_K_EXP: { const double r2 = d * d * L.mvec[0]; return exp(-sqrt(r2)); }
    case BGP_K_RATIONAL_QUADRATIC: { const double r2 = d * d * L.mvec[0]; return pow(1 + 0.5 * r2 / L.rp[0], -L.rp[0]); }
    case BGP_K_EXP_SINE2: { const double s = sin(d * L.rp[0]); return exp(-L.p[0] * s * s); }
    case BGP_K_COSINE: return cos(d * L.rp[0]);
    case BGP_K_CONSTANT: return L.rp[0];
  }
  return 0.0;
}
__device__ __forceinline__ double kernel_value_1d(const DevProgram& P, double d) {
  double s0 = 0, s1 = 0, s2 = 0, s3 = 0, s4 = 0, s5 = 0, s6 = 0, s7 = 0;
  const int n = P.n_nodes;
  for (int i = 0; i < n; ++i) {
    const int c = P.code[i];
    if (c >= 0) {
      const double v = leaf_value_1d(P.leaf[c], d);
      s7 = s6; s6 = s5; s5 = s4; s4 = s3; s3 = s2; s2 = s1; s1 = s0; s0 = v;
    } else {
      s0 = (c == -1) ? (s1 + s0) : (s1 * s0);
      s1 = s2; s2 = s3; s3 = s4; s4 = s5; s5 = s6; s6 = s7;
    }
  }
  return s0;
}

// k(x1, x2): postfix interpreter with a shift-register operand stack (no dynamically indexed local memory).
// P lives in shared memory; x1/x2 point at `ndim` doubles (shared, global or local).
__device__ __forceinline__ double kernel_value(const DevProgram& P, const double* x1, const double* x2) {
  if (P.flags & BGP_FLAG_FAST1D) return kernel_value_1d(P, x1[0] - x2[0]);
  double s0 = 0, s1 = 0, s2 = 0, s3 = 0, s4 = 0, s5 = 0, s6 = 0, s7 = 0;
  const int n = P.n_nodes;
  for (int i = 0; i < n; ++i) {
    const int c = P.code[i];
    if (c >= 0) {
      const double v = leaf_value(P.leaf[c], x1, x2);
      s7 = s6; s6 = s5; s5 = s4; s4 = s3; s3 = s2; s2 = s1; s1 = s0; s0 = v;
    } else {
      s0 = (c == -1) ? (s1 + s0) : (s1 * s0);  // kernels.h:78-80 | 114-116
      s1 = s2; s2 = s3; s3 = s4; s4 = s5; s5 = s6; s6 = s7;
    }
  }
  return s0;
}

struct GenericKernelFn {
  const DevProgram* P;
  __device__ __forceinline__ double operator()(const double* x1, const double* x2) const { return kernel_value(*P, x1, x2); }
};
// run `body(fn)` with the evaluator specialised for the program's shape
#define BGP_DISPATCH_SHAPE(P, BODY)                                                                   \
  switch ((P).shape) {                                                                                \
    case BGP_SHAPE_EXPSQ: { ScaledProfile1D<BGP_SHAPE_EXPSQ> fn{(P).sc, (P).sm}; BODY; } break;       \
    case BGP_SHAPE_M32: { ScaledProfile1D<BGP_SHAPE_M32> fn{(P).sc, (P).sm}; BODY; } break;           \
    case BGP_SHAPE_M52: { ScaledProfile1D<BGP_SHAPE_M52> fn{(P).sc, (P).sm}; BODY; } break;           \
    case BGP_SHAPE_EXP: { ScaledProfile1D<BGP_SHAPE_EXP> fn{(P).sc, (P).sm}; BODY; } break;           \
    default: { GenericKernelFn fn{&(P)}; BODY; } break;                                               \
  }
// host side: call FN<SHAPE>(args...) for the runtime shape (every shape, incl. the two-term ones)
#define BGP_SHAPE_SWITCH(shape, CALL)                                                                 \
  switch (shape) {                                                                                    \
    case BGP_SHAPE_EXPSQ: { constexpr int SHAPE = BGP_SHAPE_EXPSQ; CALL; } break;                     \
    case BGP_SHAPE_M32: { constexpr int SHAPE = BGP_SHAPE_M32; CALL; } break;                         \
    case BGP_SHAPE_M52: { constexpr int SHAPE = BGP_SHAPE_M52; CALL; } break;                         \
    case BGP_SHAPE_EXP: { constexpr int SHAPE = BGP_SHAPE_EXP; CALL; } break;                         \
    case BGP_SHAPE_SUM_EXPSQ_ES2: { constexpr int SHAPE = BGP_SHAPE_SUM_EXPSQ_ES2; CALL; } break;     \
    case BGP_SHAPE_SUM_M32_ES2: { constexpr int SHAPE = BGP_SHAPE_SUM_M32_ES2; CALL; } break;         \
    case BGP_SHAPE_PROD_EXPSQ_ES2: { constexpr int SHAPE = BGP_SHAPE_PROD_EXPSQ_ES2; CALL; } break;   \
    case BGP_SHAPE_PROD_M32_ES2: { constexpr int SHAPE = BGP_SHAPE_PROD_M32_ES2; CALL; } break;       \
    default: { constexpr int SHAPE = BGP_SHAPE_GENERIC; CALL; } break;                                \
  }

// evaluator object of a shape, built inside a kernel: the interpreter needs the staged program, the rest only scalars
template <int SHAPE>
struct ShapeEval {
  using type = ScaledProfile1D<SHAPE>;
  static __device__ __forceinline__ type make(const DevProgram* /*staged*/, const DevProgram* g) { return type(*g); }
};
template <>
struct ShapeEval<BGP_SHAPE_GENERIC> {
  using type = GenericKernelFn;
  static __device__ __forceinline__ type make(const DevProgram* staged, const DevProgram* /*g*/) { return type{staged}; }
};

// value + hyper-parameter gradient (kernels.h:81-94 Sum, 117-139 Product, per-leaf gradient() methods).
// grad has n_params_total entries; entries with which[i]==0 are 0.  Not on the log-likelihood hot path.
__device__ inline double kernel_value_grad(const DevProgram& P, const double* x1, const double* x2,
                                           const unsigned* which, double* grad) {
  double val[BGP_STACK];
  int lo[BGP_STACK], hi[BGP_STACK];
  int sp = 0;
  for (int i = 0; i < P.n_nodes; ++i) {
    const int c = P.code[i];
    if (c >= 0) {
      const DevLeaf& L = P.leaf[c];
      const int np = L.n_params + L.n_metric, off = L.param_off;
      for (int q = 0; q < np; ++q) grad[off + q] = 0.0;
      double v;
      if (L.metric_type != BGP_METRIC_NONE) {
        if (L.blocked && out_of_block(L, x1, x2)) {
          v = 0.0;
        } else {
          bool any = false;
          for (int q = L.n_params; q < np; ++q) any |= (which[off + q] != 0);
          double r2;
          if (any) {
            double mg[BGP_MAX_METRIC];
            r2 = metric_r2_grad(L, x1, x2, mg);
            const double rg = radial_gradient(L, r2);
            for (int q = 0; q < L.n_metric; ++q) grad[off + L.n_params + q] = mg[q] * rg;
          } else {
            r2 = metric_r2(L, x1, x2);
          }
          if (L.kernel_type == BGP_K_RATIONAL_QUADRATIC && which[off]) {  // kernels.h:446-452
            const double a = L.rp[0], t1 = 1.0 + 0.5 * r2 / a, t2 = 2.0 * a * t1;
            grad[off] = a * pow(t1, -a) * (r2 / t2 - log(t1));
          }
          if (L.kernel_type >= BGP_K_USER0)  // own hyper-parameters of a stationary user kernel (kernels/*.yml grad.<param>)
            for (int q = 0; q < L.n_params; ++q)
              if (which[off + q]) grad[off + q] = user::radial_param_gradient(L.kernel_type - BGP_K_USER0, q, r2, L.p, L.rp);
          v = radial_value(L, r2);
        }
      } else {
        v = 0.0;
        for (int a = 0; a < L.naxes; ++a) v += axis_value(L, x1[L.axes[a]], x2[L.axes[a]]);
        for (int q = 0; q < L.n_params; ++q) {
          if (!which[off + q]) continue;
          double g = 0.0;
          for (int a = 0; a < L.naxes; ++a) g += axis_param_gradient(L, q, x1[L.axes[a]], x2[L.axes[a]]);
          grad[off + q] = g;
        }
      }
      val[sp] = v; lo[sp] = off; hi[sp] = off + np; sp++;
    } else if (c == -1) {
      sp--; val[sp - 1] += val[sp]; hi[sp - 1] = hi[sp];
    } else {
      sp--;
      const double k1 = val[sp - 1], k2 = val[sp];
      for (int q = lo[sp - 1]; q < hi[sp - 1]; ++q) grad[q] *= k2;
      for (int q = lo[sp]; q < hi[sp]; ++q) grad[q] *= k1;
      val[sp - 1] = k1 * k2; hi[sp - 1] = hi[sp];
    }
  }
  for (int q = 0; q < P.n_params_total; ++q) if (!which[q]) grad[q] = 0.0;
  return val[0];
}

// ---- gradients with respect to the input coordinates (kernel_interface.cpp:127-157) ---------------------------------
// side 1: d k / d x1, side 2: d k / d x2.  Needs ndim <= BGP_MAX_DIM.
// EXACT = false is the reference's x-gradient, which get_x1_gradient / get_x2_gradient reproduce: for a general metric
// M = L L^T it returns L^-1 r (metrics.h:233-246), not the derivative of r^T M^-1 r, which needs L^-T L^-1 r.
// EXACT = true applies that backward substitution as well: the true derivative for every metric (GP.grad_predict).
__device__ inline double axis_x_gradient(const DevLeaf& L, int side, double x1, double x2) {
  switch (L.kernel_type) {
    case BGP_K_LINEAR:
      if (L.p[1] == 0.0) return 0.0;
      return (side == 1 ? x2 : x1) * L.p[1] * pow(x1 * x2, L.p[1] - 1.0) * L.rp[0];
    case BGP_K_LOCAL_GAUSSIAN: {
      const double d1 = x1 - L.p[0], d2 = x2 - L.p[0];
      return -2.0 * exp(-(d1 * d1 + d2 * d2) * L.rp[0]) * (side == 1 ? d1 : d2) * L.rp[0];
    }
    case BGP_K_COSINE: return (side == 1 ? -L.rp[0] : L.rp[0]) * sin(L.rp[0] * (x1 - x2));
    case BGP_K_EXP_SINE2: {
      const double d = x1 - x2, s = sin(d * L.rp[0]);
      const double g = exp(-L.p[0] * s * s) * L.rp[0] * L.p[0] * sin(2.0 * L.rp[0] * d);
      return side == 1 ? -g : g;
    }
    case BGP_K_POLYNOMIAL:
      if (L.p[1] == 0.0) return 0.0;
      return (side == 1 ? x2 : x1) * L.p[1] * pow(x1 * x2 + L.rp[0], L.p[1] - 1.0);
    case BGP_K_DOT_PRODUCT: return side == 1 ? x2 : x1;
  }
  if (L.kernel_type >= BGP_K_USER0) return user::axis_x_gradient(L.kernel_type - BGP_K_USER0, side, x1, x2, L.p, L.rp);
  return 0.0;
}
template <bool EXACT = false>
__device__ inline void leaf_x_gradient(const DevLeaf& L, int ndim, int side, const double* x1, const double* x2,
                                       double* grad) {
  for (int i = 0; i < ndim; ++i) grad[i] = 0.0;
  if (L.metric_type != BGP_METRIC_NONE) {  // e.g. kernels.h:1953-2003
    if (L.blocked && out_of_block(L, x1, x2)) return;
    const double r2grad = 2.0 * radial_gradient(L, metric_r2(L, x1, x2));
    if (L.metric_type == BGP_METRIC_ISOTROPIC) {        // metrics.h:93-99
      for (int i = 0; i < L.naxes; ++i) { const int j = L.axes[i]; grad[j] = L.mvec[0] * (x1[j] - x2[j]); }
    } else if (L.metric_type == BGP_METRIC_AXIS_ALIGNED) {  // metrics.h:133-138
      for (int i = 0; i < L.naxes; ++i) { const int j = L.axes[i]; grad[j] = L.mvec[i] * (x1[j] - x2[j]); }
    } else {                                              // metrics.h:233-246: forward substitution only
      double r[BGP_MAX_DIM];
      const int n = L.naxes;
      int k = 0;
      for (int i = 0; i < n; ++i) {
        double b = x1[L.axes[i]] - x2[L.axes[i]];
        for (int j = 0; j < i; ++j, ++k) b -= L.mvec[k] * r[j];
        b *= L.mvec[k++];
        r[i] = b;
      }
      if (EXACT) {  // r <- L^-T r, the backward substitution of metric_r2_grad (metrics.h:153-164)
        const int k0 = (n + 1) * n / 2;
        for (int i = n - 1; i >= 0; --i) {
          int kk = k0 - n + i;
          for (int j = n - 1; j > i; --j) {
            r[i] -= L.mvec[kk] * r[j];
            kk -= j;
          }
          r[i] *= L.mvec[kk];
        }
      }
      for (int i = 0; i < n; ++i) grad[L.axes[i]] = r[i];
    }
    for (int i = 0; i < ndim; ++i) grad[i] *= (side == 1 ? r2grad : -r2grad);
    return;
  }
  for (int i = 0; i < L.naxes; ++i) { const int j = L.axes[i]; grad[j] = axis_x_gradient(L, side, x1[j], x2[j]); }
}
// Sum: kernels.h:94-108, Product: kernels.h:140-162
template <bool EXACT = false>
__device__ inline void kernel_x_gradient(const DevProgram& P, int side, const double* x1, const double* x2, double* out) {
  double g[BGP_STACK][BGP_MAX_DIM];
  double val[BGP_STACK];
  int sp = 0;
  const int nd = P.ndim;
  for (int i = 0; i < P.n_nodes; ++i) {
    const int c = P.code[i];
    if (c >= 0) {
      leaf_x_gradient<EXACT>(P.leaf[c], nd, side, x1, x2, g[sp]);
      val[sp] = leaf_value(P.leaf[c], x1, x2);
      sp++;
    } else {
      sp--;
      if (c == -1) {
        for (int q = 0; q < nd; ++q) g[sp - 1][q] = g[sp - 1][q] + g[sp][q];
        val[sp - 1] += val[sp];
      } else {
        const double k1 = val[sp - 1], k2 = val[sp];
        for (int q = 0; q < nd; ++q) g[sp - 1][q] = k2 * g[sp - 1][q] + k1 * g[sp][q];
        val[sp - 1] = k1 * k2;
      }
    }
  }
  for (int q = 0; q < nd; ++q) out[q] = g[0][q];
}

// d k(x1, x2) / d x1 on GP.grad_predict's hot path (kmat_ops.cu: kmat_x1_grad_matvec_kernel).  The one-term 1-D
// shapes of BGP_DISPATCH_SHAPE,  c * f(m d^2),  get  c * f'(r2) * 2 m d  with f' the radial_gradient of the profile (the
// far-pair cutoffs of profile_value, where f' underflows to 0 as well); every other program runs the interpreter with
// the exact metric derivative.  NDMAX: the entries of g an evaluator writes (ndim of it).
template <int PROFILE>
__device__ __forceinline__ double profile_gradient(double r2) {
  if (PROFILE == BGP_SHAPE_EXPSQ) return (r2 > 1490.4) ? 0.0 : -0.5 * exp(-0.5 * r2);
  if (PROFILE == BGP_SHAPE_M32) {
    if (r2 > 185200.0 && r2 <= DBL_MAX) return 0.0;
    const double r = sqrt(3.0 * r2);
    return -3.0 * 0.5 * exp(-r);
  }
  if (PROFILE == BGP_SHAPE_M52) {
    if (r2 > 111100.0 && r2 <= DBL_MAX) return 0.0;
    const double r = sqrt(5.0 * r2);
    return -5 * (1 + r) * exp(-r) / 6.0;
  }
  if (r2 < 2.220446049250313e-16 || r2 > 555400.0) return 0.0;  // Exp: a coincident pair has a finite (zero) gradient
  const double r = sqrt(r2);
  return -0.5 * exp(-r) / r;
}
template <int SHAPE>
struct ScaledProfileGrad1D {
  static constexpr int NDMAX = 1;
  double c, m;
  __device__ __forceinline__ void operator()(const double* x1, const double* x2, double* g) const {
    const double d = x1[0] - x2[0];
    g[0] = c * (2.0 * profile_gradient<SHAPE>(d * d * m)) * (m * d);
  }
};
struct GenericX1GradFn {
  static constexpr int NDMAX = BGP_MAX_DIM;
  const DevProgram* P;
  __device__ __forceinline__ void operator()(const double* x1, const double* x2, double* g) const {
    kernel_x_gradient<true>(*P, 1, x1, x2, g);
  }
};
template <int SHAPE>
struct X1GradEval {
  using type = ScaledProfileGrad1D<SHAPE>;
  static __device__ __forceinline__ type make(const DevProgram* staged) { return type{staged->sc, staged->sm}; }
};
template <>
struct X1GradEval<BGP_SHAPE_GENERIC> {
  using type = GenericX1GradFn;
  static __device__ __forceinline__ type make(const DevProgram* staged) { return type{staged}; }
};

#endif  // __CUDACC__

}  // namespace bgp
