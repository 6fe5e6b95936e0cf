// amg.cu — algebraic multigrid of an assembled sparse matrix, the preconditioners of GMRES on the sparse route that the tutorial
// builds with AlgebraicMultigrid.jl (`KrylovJL_GMRES(precs = ...)` with `aspreconditioner(ruge_stuben(W))` or
// `aspreconditioner(smoothed_aggregation(W))` and Jacobi smoothing, docs/src/tutorials/large_systems.md:244-316).  Two coarsenings
// share one hierarchy, one refresh of the Galerkin products and one V-cycle:
//
//   * classical Ruge-Stueben (DESIGN.md §4h): classical strength (j strongly influences i when |a_ij| >= theta max_{k != i}
//     |a_ik|), the Ruge-Stueben first-pass C/F splitting, sign-split direct interpolation;
//   * smoothed aggregation (DESIGN.md §4i): symmetric strength, a distance-2 maximal independent set as aggregate roots, a
//     piecewise-constant tentative prolongator T and P = T - (omega_P / rho) D^-1 A T, rho the Gershgorin bound of D^-1 A.
//
// Both take Galerkin coarse operators A_{l+1} = R A_l P with R = P' stored explicitly and the coarsest level's explicit inverse.
//
// Where the work runs:
//   * rebuild (once per solve): every pattern comes from the device sparse product below (expand, stable radix sort, compress),
//     which also gives the pair lists of A P and R (A P) and, on a (column, row) key, the transpose R = P' with its gather map.
//     Ruge-Stueben keeps strength and the splitting on the host, so each coarse level's values come down to choose the next
//     splitting; smoothed aggregation runs every step on the device and reads back sizes only;
//   * refresh (device, every later fresh Jacobian): gather, inverse diagonals, P's values (interpolation weights, or rho, A T
//     and the smoothing), R = P' by a gather, A P and R (A P) by one pair-list product kernel, the coarsest inverse by getrf /
//     getrs.  Every sum runs in a fixed order and there is no floating-point atomic: a refresh is bit-reproducible, and a
//     rebuild gives the same bits;
//   * apply: one V-cycle, damped Jacobi (the first pre-sweep from x = 0 is x = omega D^-1 b), residual, restriction, prolongation
//     and the coarsest GEMV, captured once per rebuild into a CUDA graph (a refresh writes values in place, so the graph stays valid).
#include "common.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <algorithm>
#include <climits>
#include <cmath>
#include <queue>
#include <vector>

namespace {
constexpr int AT = 256;
constexpr int64_t AMG_DENSE_CAP = 4096;  // largest coarsest level that gets an explicit dense inverse
enum { AMG_RS = 0, AMG_SA = 1 };
// why coarsening stopped: at max_coarse or max_levels, or stalled: a level with no coarse point / aggregate (no point has a
// strong connection), or one per unknown (no reduction).  The second is a guard that no input reaches: with any strong
// connection the Ruge-Stueben pass makes its first pick's dependents F, and a root's graph neighbours are never roots
enum { AMG_STOP_SIZE = 0, AMG_STOP_NONE = 1, AMG_STOP_ALL = 2 };

// one level of the hierarchy on the device; P, R and the product lists exist on every level but the coarsest
struct AmgLevel {
  int32_t n = 0, nnz = 0;                    // A_l
  int32_t *rowptr = nullptr, *col = nullptr, *diag = nullptr;
  double *val = nullptr, *dinv = nullptr;
  int32_t pnnz = 0;                          // P_l: n x n_{l+1}
  int32_t *prowptr = nullptr, *pcol = nullptr, *pmap = nullptr;  // RS: pmap = P position -> A_l position (-1 on C rows)
  double* pval = nullptr;
  int32_t *rrowptr = nullptr, *rcol = nullptr, *rmap = nullptr;  // R = P': rmap = R position -> P position
  double* rval = nullptr;
  int32_t apnnz = 0;                         // A_l P_l: values only (the pair lists address them)
  double* apval = nullptr;
  int32_t *ap_ptr = nullptr, *ap_x = nullptr, *ap_y = nullptr;   // AP[q] = sum_t A[ap_x[t]] P[ap_y[t]], t in [ap_ptr[q], ap_ptr[q+1])
  int32_t *ac_ptr = nullptr, *ac_x = nullptr, *ac_y = nullptr;   // A_{l+1}[q] = sum_t R[ac_x[t]] AP[ac_y[t]]
  // SA: the tentative prolongator (one entry per aggregated row, fixed at rebuild), A_l T_l on P_l's pattern, rho as double bits
  int32_t tnnz = 0;
  int32_t *trowptr = nullptr, *tcol = nullptr;
  double *tval = nullptr, *atval = nullptr;
  int32_t *at_ptr = nullptr, *at_x = nullptr, *at_y = nullptr;   // AT[q] = sum_t A[at_x[t]] T[at_y[t]], q a P position
  unsigned long long* rho = nullptr;
  double *x = nullptr, *x2 = nullptr, *b = nullptr, *r = nullptr;
};

// host CSR of one Ruge-Stueben level while the hierarchy is built
struct HostLevel {
  int32_t n = 0;
  std::vector<int32_t> rowptr, col;
  std::vector<double> val;
};
}  // namespace

struct b200_amg {
  b200_ctx* ctx;
  int64_t n, nnz;
  int method = AMG_RS;
  b200_amg_opts o;                           // SA handles: the shared fields of b200_sa_opts
  double smooth_omega = 0.0;                 // SA: omega_P
  std::vector<int32_t> rowptr0, col0, map0;  // level-0 CSR view of the caller's CSC pattern
  int32_t* d_map0 = nullptr;
  std::vector<AmgLevel> lev;
  std::vector<void*> owned;                  // device allocations of the current hierarchy
  double *d_dense = nullptr, *d_ainv = nullptr;  // coarsest level: LU workspace, explicit inverse
  int64_t* d_ipiv = nullptr;
  int32_t* d_info = nullptr;
  int built = 0, refreshed = 0;
  int stall = 0;                             // why the last rebuild stopped coarsening (AMG_STOP_*)
  cudaGraphExec_t gexec = nullptr;
  bool graph_unavailable = false;
  int64_t glaunches = 0;
  double* gres = nullptr;
};

namespace {
// ---------------------------------------------------------------- device refresh
__global__ void __launch_bounds__(AT) amg_gather_kernel(int32_t nnz, const int32_t* __restrict__ map, const double* __restrict__ src, double* __restrict__ dst) {
  const int32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q < nnz) dst[q] = src[map[q]];
}

// direct interpolation weights of every row (one thread per row); C rows hold their unit entry.  *info = level + 1 when a
// denominator a_ii (after the positive lumping) is zero or not finite
__global__ void __launch_bounds__(AT) amg_interp_kernel(int32_t n, const int32_t* __restrict__ rowptr, const int32_t* __restrict__ col,
                                                        const int32_t* __restrict__ diag, const double* __restrict__ a, const int32_t* __restrict__ prowptr,
                                                        const int32_t* __restrict__ pmap, double* __restrict__ p, int32_t level, int32_t* info) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t p0 = prowptr[i], p1 = prowptr[i + 1];
  if (p1 == p0) return;                       // isolated F point: empty row
  if (pmap[p0] < 0) { p[p0] = 1.0; return; }  // C point
  double an = 0.0, ap = 0.0, sn = 0.0, sp = 0.0;
  for (int32_t q = rowptr[i]; q < rowptr[i + 1]; ++q) {
    if (col[q] == i) continue;
    const double v = a[q];
    if (v < 0.0) an += v; else if (v > 0.0) ap += v;
  }
  for (int32_t t = p0; t < p1; ++t) {
    const double v = a[pmap[t]];
    if (v < 0.0) sn += v; else if (v > 0.0) sp += v;
  }
  double d = a[diag[i]];
  const double alpha = sn != 0.0 ? an / sn : 0.0;
  double beta = 0.0;
  if (sp == 0.0) d += ap; else beta = ap / sp;
  if (d == 0.0 || !isfinite(d)) atomicMin(info, level + 1);
  for (int32_t t = p0; t < p1; ++t) {
    const double v = a[pmap[t]];
    p[t] = -((v < 0.0 ? alpha : beta) * v) / d;
  }
}

// out[q] = sum over the pair list of q of X[x] Y[y], in list order (both Galerkin products: A P, then R (A P))
__global__ void __launch_bounds__(AT) amg_pair_product_kernel(int32_t nout, const int32_t* __restrict__ ptr, const int32_t* __restrict__ xi,
                                                              const int32_t* __restrict__ yi, const double* __restrict__ X, const double* __restrict__ Y,
                                                              double* __restrict__ out) {
  const int32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nout) return;
  double s = 0.0;
  for (int32_t t = ptr[q]; t < ptr[q + 1]; ++t) s = fma(X[xi[t]], Y[yi[t]], s);
  out[q] = s;
}

__global__ void __launch_bounds__(AT) amg_dinv_kernel(int32_t n, const int32_t* __restrict__ diag, const double* __restrict__ a, double* __restrict__ dinv,
                                                      int32_t level, int32_t* info) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double d = a[diag[i]];
  if (d == 0.0 || !isfinite(d)) atomicMin(info, level + 1);
  dinv[i] = 1.0 / d;
}

// the coarsest level as a dense column-major matrix (pre-zeroed), and the identity its inverse is solved from
__global__ void __launch_bounds__(AT) amg_densify_kernel(int32_t n, const int32_t* __restrict__ rowptr, const int32_t* __restrict__ col,
                                                         const double* __restrict__ a, double* __restrict__ D) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int32_t q = rowptr[i]; q < rowptr[i + 1]; ++q) D[(int64_t)col[q] * n + i] = a[q];
}
__global__ void __launch_bounds__(AT) amg_identity_kernel(int64_t n, double* __restrict__ E) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n * n) E[k] = (k % n == k / n) ? 1.0 : 0.0;
}

// ---------------------------------------------------------------- apply
__global__ void __launch_bounds__(AT) amg_jacobi0_kernel(int32_t n, double omega, const double* __restrict__ dinv, const double* __restrict__ b, double* __restrict__ x) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] = omega * dinv[i] * b[i];
}
// jac = 0: r = b - A x;  jac = 1: r = x + omega D^-1 (b - A x)  (the fused residual-and-Jacobi sweep; r != x)
__global__ void __launch_bounds__(AT) amg_residual_kernel(int32_t n, const int32_t* __restrict__ rowptr, const int32_t* __restrict__ col,
                                                          const double* __restrict__ a, const double* __restrict__ x, const double* __restrict__ b,
                                                          int jac, double omega, const double* __restrict__ dinv, double* __restrict__ r) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double s = 0.0;
  for (int32_t q = rowptr[i]; q < rowptr[i + 1]; ++q) s = fma(a[q], x[col[q]], s);
  const double res = b[i] - s;
  r[i] = jac ? fma(omega * dinv[i], res, x[i]) : res;
}
// add = 0: y = M x;  add = 1: y += M x  (restriction with R, prolongation with P)
__global__ void __launch_bounds__(AT) amg_spmv_kernel(int32_t n, const int32_t* __restrict__ rowptr, const int32_t* __restrict__ col,
                                                      const double* __restrict__ m, const double* __restrict__ x, int add, double* __restrict__ y) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double s = 0.0;
  for (int32_t q = rowptr[i]; q < rowptr[i + 1]; ++q) s = fma(m[q], x[col[q]], s);
  y[i] = add ? y[i] + s : s;
}

// ---------------------------------------------------------------- device sparse product with pair lists
// Z = X Y by expand-sort-compress.  One thread per X row writes its terms (row, Y column) with payload (X position, Y position)
// in the order X positions ascending, then Y positions ascending; a stable radix sort on the packed key groups equal entries
// with their terms in that order; run heads scanned give Z's pattern.  With Y = I (yrowptr null) and the key (column, row) the
// same steps give X' with its gather map (Z's rows are X's columns, the pair list's x the X position of each entry).
__global__ void __launch_bounds__(AT) sp_count_kernel(int32_t nx, const int32_t* __restrict__ xrowptr, const int32_t* __restrict__ xcol,
                                                      const int32_t* __restrict__ yrowptr, int64_t* __restrict__ cnt) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > nx) return;
  int64_t c = 0;
  if (i < nx)
    for (int32_t q = xrowptr[i]; q < xrowptr[i + 1]; ++q) c += yrowptr ? yrowptr[xcol[q] + 1] - yrowptr[xcol[q]] : 1;
  cnt[i] = c;
}

__global__ void __launch_bounds__(AT) sp_expand_kernel(int32_t nx, const int32_t* __restrict__ xrowptr, const int32_t* __restrict__ xcol,
                                                       const int32_t* __restrict__ yrowptr, const int32_t* __restrict__ ycol, uint64_t p, int transpose,
                                                       const int64_t* __restrict__ off, uint64_t* __restrict__ key, int32_t* __restrict__ idx,
                                                       int32_t* __restrict__ tx, int32_t* __restrict__ ty) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nx) return;
  int64_t o = off[i];
  for (int32_t q = xrowptr[i]; q < xrowptr[i + 1]; ++q) {
    const int32_t j = xcol[q];
    const int32_t t0 = yrowptr ? yrowptr[j] : j, t1 = yrowptr ? yrowptr[j + 1] : j + 1;
    for (int32_t t = t0; t < t1; ++t, ++o) {
      const uint64_t c = yrowptr ? (uint64_t)ycol[t] : (uint64_t)j;
      key[o] = transpose ? c * (uint64_t)nx + (uint64_t)i : (uint64_t)i * p + c;
      idx[o] = (int32_t)o; tx[o] = q; ty[o] = t;
    }
  }
}

__global__ void __launch_bounds__(AT) sp_heads_kernel(int32_t nt, const uint64_t* __restrict__ key, int32_t* __restrict__ head) {
  const int32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k <= nt) head[k] = k < nt && (k == 0 || key[k] != key[k - 1]);
}

// hs: exclusive scan of the heads (hs[nt] = Z's nnz).  Row r of Z starts at the first output of the first term with row >= r
__global__ void __launch_bounds__(AT) sp_compress_kernel(int32_t nt, int32_t nrows, uint64_t div, const uint64_t* __restrict__ key,
                                                         const int32_t* __restrict__ idx, const int32_t* __restrict__ hs, const int32_t* __restrict__ tx,
                                                         const int32_t* __restrict__ ty, int32_t* __restrict__ rowptr, int32_t* __restrict__ col,
                                                         int32_t* __restrict__ ptr, int32_t* __restrict__ px, int32_t* __restrict__ py) {
  const int32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k > nt) return;
  if (k < nt) {
    const int32_t s = idx[k];
    px[k] = tx[s];
    if (py) py[k] = ty[s];
    if (k == 0 || key[k] != key[k - 1]) {
      col[hs[k]] = (int32_t)(key[k] % div);
      if (ptr) ptr[hs[k]] = k;
    }
  } else if (ptr) {
    ptr[hs[nt]] = nt;
  }
  const int64_t r1 = k < nt ? (int64_t)(key[k] / div) : nrows;
  const int64_t r0 = k > 0 ? (int64_t)(key[k - 1] / div) : -1;
  for (int64_t r = r0 + 1; r <= r1; ++r) rowptr[r] = hs[k];
}

// ---------------------------------------------------------------- smoothed aggregation
enum : uint32_t { SA_OUT = 0, SA_UNDECIDED = 1, SA_IN = 2 };

// the node priority: a bijection of 32-bit integers, so (h, i) orders as h alone and a node is known by its h
__device__ __forceinline__ uint32_t sa_hash(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
  return x;
}

// the strength graph, symmetric: j is a neighbour of i when the entry (i, j) or (j, i) is strong; the second half walks A' (its
// rows are A's columns, tmap the A position of each entry)
struct SaGraph {
  const int32_t *rowptr, *col, *trowptr, *tcol, *tmap;
  const uint8_t* strong;
  template <class F>
  __device__ __forceinline__ void each(int32_t i, F f) const {
    for (int32_t q = rowptr[i]; q < rowptr[i + 1]; ++q)
      if (strong[q]) f(col[q]);
    for (int32_t t = trowptr[i]; t < trowptr[i + 1]; ++t)
      if (strong[tmap[t]]) f(tcol[t]);
  }
};

__global__ void __launch_bounds__(AT) amg_diag_kernel(int32_t n, const int32_t* __restrict__ rowptr, const int32_t* __restrict__ col, int32_t* __restrict__ diag) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int32_t d = -1;
  for (int32_t q = rowptr[i]; q < rowptr[i + 1]; ++q)
    if (col[q] == i) d = q;
  diag[i] = d;
}

// j != i is strong when a_ij != 0 and |a_ij| >= theta sqrt(|a_ii| |a_jj|)
__global__ void __launch_bounds__(AT) sa_strength_kernel(int32_t n, const int32_t* __restrict__ rowptr, const int32_t* __restrict__ col,
                                                         const int32_t* __restrict__ diag, const double* __restrict__ a, double theta, uint8_t* __restrict__ strong) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double di = fabs(a[diag[i]]);
  for (int32_t q = rowptr[i]; q < rowptr[i + 1]; ++q) {
    const int32_t j = col[q];
    const double v = a[q];
    strong[q] = j != i && v != 0.0 && fabs(v) >= theta * sqrt(di * fabs(a[diag[j]]));
  }
}

// key = (state, h): isolated nodes start OUT, every other node UNDECIDED
__global__ void __launch_bounds__(AT) sa_mis_init_kernel(int32_t n, SaGraph g, uint64_t* __restrict__ key) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  bool edge = false;
  g.each(i, [&](int32_t) { edge = true; });
  key[i] = ((uint64_t)(edge ? SA_UNDECIDED : SA_OUT) << 32) | sa_hash((uint32_t)i);
}

// one max-propagation: out[i] = the largest key among i and its neighbours
__global__ void __launch_bounds__(AT) sa_max_kernel(int32_t n, SaGraph g, const uint64_t* __restrict__ in, uint64_t* __restrict__ out) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t m = in[i];
  g.each(i, [&](int32_t j) { m = max(m, in[j]); });
  out[i] = m;
}

// an undecided node that is its own distance-2 maximum joins the set; one whose distance-2 maximum is in the set leaves
__global__ void __launch_bounds__(AT) sa_mis_update_kernel(int32_t n, uint64_t* __restrict__ key, const uint64_t* __restrict__ m2, int32_t* __restrict__ undecided) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t k = key[i];
  if ((k >> 32) != SA_UNDECIDED) return;
  if (m2[i] == k) key[i] = ((uint64_t)SA_IN << 32) | (k & 0xffffffffu);
  else if ((m2[i] >> 32) == SA_IN) key[i] = ((uint64_t)SA_OUT << 32) | (k & 0xffffffffu);
  else atomicAdd(undecided, 1);
}

// flag[i] = i is a root (flag[n] = 0: the exclusive scan's last entry counts the roots)
__global__ void __launch_bounds__(AT) sa_root_flag_kernel(int32_t n, const uint64_t* __restrict__ key, int32_t* __restrict__ flag) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i <= n) flag[i] = i < n && (key[i] >> 32) == SA_IN;
}

// pass 1: a root takes its number, every other node the adjacent root of largest h (or -1)
__global__ void __launch_bounds__(AT) sa_pass1_kernel(int32_t n, SaGraph g, const uint64_t* __restrict__ key, const int32_t* __restrict__ rid, int32_t* __restrict__ agg) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if ((key[i] >> 32) == SA_IN) { agg[i] = rid[i]; return; }
  uint64_t best = 0;
  int32_t a = -1;
  g.each(i, [&](int32_t j) {
    if ((key[j] >> 32) == SA_IN && (a < 0 || key[j] > best)) { best = key[j]; a = rid[j]; }
  });
  agg[i] = a;
}

// pass 2: a node still unassigned joins the neighbour of largest h among those assigned after pass 1
__global__ void __launch_bounds__(AT) sa_pass2_kernel(int32_t n, SaGraph g, const int32_t* __restrict__ agg1, int32_t* __restrict__ agg2) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int32_t a = agg1[i];
  if (a < 0) {
    uint32_t best = 0;
    g.each(i, [&](int32_t j) {
      const uint32_t h = sa_hash((uint32_t)j);
      if (agg1[j] >= 0 && (a < 0 || h > best)) { best = h; a = agg1[j]; }
    });
  }
  agg2[i] = a;
}

// flag[i] = i is aggregated (flag[n] = 0); the exclusive scan is T's rowptr
__global__ void __launch_bounds__(AT) sa_tflag_kernel(int32_t n, const int32_t* __restrict__ agg, int32_t* __restrict__ flag) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i <= n) flag[i] = i < n && agg[i] >= 0;
}
__global__ void __launch_bounds__(AT) sa_tcol_kernel(int32_t n, const int32_t* __restrict__ agg, const int32_t* __restrict__ trowptr, int32_t* __restrict__ tcol) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && agg[i] >= 0) tcol[trowptr[i]] = agg[i];
}

// ||b restricted to aggregate a||, summed over its members in node order (mrowptr / mcol: T', one row per aggregate)
__global__ void __launch_bounds__(AT) sa_norm_kernel(int32_t na, const int32_t* __restrict__ mrowptr, const int32_t* __restrict__ mcol, const double* __restrict__ b,
                                                     double* __restrict__ nrm) {
  const int32_t a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= na) return;
  double s = 0.0;
  for (int32_t t = mrowptr[a]; t < mrowptr[a + 1]; ++t) s = __dadd_rn(s, __dmul_rn(b[mcol[t]], b[mcol[t]]));
  nrm[a] = sqrt(s);
}
__global__ void __launch_bounds__(AT) sa_tval_kernel(int32_t n, const int32_t* __restrict__ trowptr, const int32_t* __restrict__ tcol, const double* __restrict__ b,
                                                     const double* __restrict__ nrm, double* __restrict__ tval) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && trowptr[i + 1] > trowptr[i]) tval[trowptr[i]] = b[i] / nrm[tcol[trowptr[i]]];
}

// rho = max_i sum_j |a_ij| / |a_ii| (the Gershgorin bound of D^-1 A), as the bits of a non-negative double under an integer max
__global__ void __launch_bounds__(AT) sa_rho_kernel(int32_t n, const int32_t* __restrict__ rowptr, const int32_t* __restrict__ diag, const double* __restrict__ a,
                                                    unsigned long long* __restrict__ rho) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double s = 0.0;
  for (int32_t q = rowptr[i]; q < rowptr[i + 1]; ++q) s += fabs(a[q]);
  atomicMax(rho, (unsigned long long)__double_as_longlong(s / fabs(a[diag[i]])));
}

// P = T - (omega_P / rho) D^-1 (A T) on A T's pattern, which holds T's
__global__ void __launch_bounds__(AT) sa_p_kernel(int32_t n, const int32_t* __restrict__ prowptr, const int32_t* __restrict__ pcol, const int32_t* __restrict__ trowptr,
                                                  const int32_t* __restrict__ tcol, const double* __restrict__ tval, const double* __restrict__ dinv,
                                                  const double* __restrict__ atv, const unsigned long long* __restrict__ rho, double omega_p, double* __restrict__ p) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const bool agg = trowptr[i + 1] > trowptr[i];
  const int32_t tc = agg ? tcol[trowptr[i]] : -1;
  const double tv = agg ? tval[trowptr[i]] : 0.0;
  const double c = omega_p / __longlong_as_double((long long)*rho) * dinv[i];
  for (int32_t q = prowptr[i]; q < prowptr[i + 1]; ++q) p[q] = fma(-c, atv[q], pcol[q] == tc ? tv : 0.0);
}

inline int blocks(int64_t n) { return (int)std::max<int64_t>(1, (n + AT - 1) / AT); }

// ---------------------------------------------------------------- host: strength and splitting (Ruge-Stueben)
// strong[q] for every CSR position q of a row
void strength(int32_t n, const std::vector<int32_t>& rowptr, const std::vector<int32_t>& col, const double* val, double theta, std::vector<char>& strong) {
  strong.assign(rowptr[n], 0);
  for (int32_t i = 0; i < n; ++i) {
    double mx = 0.0;
    for (int32_t q = rowptr[i]; q < rowptr[i + 1]; ++q)
      if (col[q] != i) mx = std::max(mx, std::fabs(val[q]));
    if (!(mx > 0.0)) continue;
    for (int32_t q = rowptr[i]; q < rowptr[i + 1]; ++q)
      strong[q] = col[q] != i && val[q] != 0.0 && std::fabs(val[q]) >= theta * mx;
  }
}

// the Ruge-Stueben first pass; cf[i] = 1 (C) or 0 (F).  A max-heap on (lambda, -i) with stale entries skipped: lambda only grows
int64_t rs_split(int32_t n, const std::vector<int32_t>& rowptr, const std::vector<int32_t>& col, const std::vector<char>& strong, std::vector<int32_t>& cf) {
  std::vector<int32_t> tptr(n + 1, 0), tcol;  // S': row j lists the points j strongly influences
  for (int32_t i = 0; i < n; ++i)
    for (int32_t q = rowptr[i]; q < rowptr[i + 1]; ++q)
      if (strong[q]) tptr[col[q] + 1]++;
  for (int32_t j = 0; j < n; ++j) tptr[j + 1] += tptr[j];
  tcol.resize(tptr[n]);
  {
    std::vector<int32_t> fill(tptr.begin(), tptr.end() - 1);
    for (int32_t i = 0; i < n; ++i)
      for (int32_t q = rowptr[i]; q < rowptr[i + 1]; ++q)
        if (strong[q]) tcol[fill[col[q]]++] = i;
  }
  enum : int8_t { U = 0, C = 1, F = 2 };
  std::vector<int8_t> st(n, U);
  std::vector<int32_t> lam(n, 0);
  std::priority_queue<std::pair<int32_t, int32_t>> heap;
  for (int32_t i = 0; i < n; ++i) {
    bool dep = false;
    for (int32_t q = rowptr[i]; q < rowptr[i + 1] && !dep; ++q) dep = strong[q];
    lam[i] = tptr[i + 1] - tptr[i];
    if (!dep && lam[i] == 0) st[i] = F;  // isolated
    else heap.push({lam[i], -i});
  }
  int64_t nc = 0;
  while (!heap.empty()) {
    const auto top = heap.top();
    heap.pop();
    const int32_t i = -top.second;
    if (st[i] != U || top.first != lam[i]) continue;
    st[i] = C;
    ++nc;
    for (int32_t t = tptr[i]; t < tptr[i + 1]; ++t) {
      const int32_t j = tcol[t];
      if (st[j] != U) continue;
      st[j] = F;
      for (int32_t q = rowptr[j]; q < rowptr[j + 1]; ++q) {
        const int32_t k = col[q];
        if (strong[q] && st[k] == U) heap.push({++lam[k], -k});
      }
    }
  }
  cf.resize(n);
  for (int32_t i = 0; i < n; ++i) cf[i] = st[i] == C;
  return nc;
}

// P's pattern: a C row holds its unit entry (pmap -1), an F row its strong C-neighbours (pmap: their A positions)
void interpolation_pattern(const HostLevel& L, const std::vector<char>& strong, const std::vector<int32_t>& cf, std::vector<int32_t>& prowptr,
                           std::vector<int32_t>& pcol, std::vector<int32_t>& pmap) {
  const int32_t n = L.n;
  std::vector<int32_t> cidx(n, -1);
  int32_t nc = 0;
  for (int32_t i = 0; i < n; ++i)
    if (cf[i]) cidx[i] = nc++;
  prowptr.assign(n + 1, 0); pcol.clear(); pmap.clear();
  for (int32_t i = 0; i < n; ++i) {
    if (cf[i]) {
      pcol.push_back(cidx[i]); pmap.push_back(-1);
    } else {
      for (int32_t q = L.rowptr[i]; q < L.rowptr[i + 1]; ++q)
        if (L.col[q] != i && strong[q] && cf[L.col[q]]) { pcol.push_back(cidx[L.col[q]]); pmap.push_back(q); }
    }
    prowptr[i + 1] = (int32_t)pcol.size();
  }
}

// ---------------------------------------------------------------- host: device memory of the setup
template <typename T>
int32_t dalloc(b200_ctx* ctx, std::vector<void*>& owner, T** p, size_t count) {
  if (cudaMalloc(p, sizeof(T) * std::max<size_t>(count, 1)) != cudaSuccess) {
    cudaGetLastError();
    *p = nullptr;
    return ctx->fail(B200_ERR_NOMEM, "AMG: the hierarchy does not fit in device memory", __FILE__, __LINE__);
  }
  owner.push_back(*p);
  return B200_OK;
}
template <typename T>
int32_t upload(b200_ctx* ctx, std::vector<void*>& owner, T** p, const std::vector<T>& h) {
  B200_TRY(dalloc(ctx, owner, p, h.size()));
  if (!h.empty()) CUDA_TRY(ctx, cudaMemcpyAsync(*p, h.data(), sizeof(T) * h.size(), cudaMemcpyHostToDevice, ctx->stream));
  return B200_OK;
}
template <typename T>
int32_t download(b200_ctx* ctx, std::vector<T>& h, const T* d, size_t count) {
  h.resize(count);
  if (count) CUDA_TRY(ctx, cudaMemcpyAsync(h.data(), d, sizeof(T) * count, cudaMemcpyDeviceToHost, ctx->stream));
  return B200_OK;
}
// transient buffers of one setup step, freed when it returns
struct Scratch {
  std::vector<void*> p;
  Scratch() = default;
  Scratch(const Scratch&) = delete;
  ~Scratch() { for (void* q : p) cudaFree(q); }
};

int32_t scan_i32(b200_ctx* ctx, const int32_t* in, int32_t* out, int64_t count) {
  Scratch s;
  size_t bytes = 0;
  CUDA_TRY(ctx, cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, count, ctx->stream));
  void* tmp = nullptr;
  B200_TRY(dalloc(ctx, s.p, (char**)&tmp, bytes));
  CUDA_TRY(ctx, cub::DeviceScan::ExclusiveSum(tmp, bytes, in, out, count, ctx->stream));
  return B200_OK;
}

// a device CSR pattern and the pair lists of a product (ptr / y null for a transpose, whose x is the gather map)
struct DevCsr { int32_t nrows = 0, nnz = 0; int32_t *rowptr = nullptr, *col = nullptr; };
struct PairLists { int32_t *ptr = nullptr, *x = nullptr, *y = nullptr; };

const char* const AMG_PRODUCT_LIMIT = "a Galerkin product has 2^31 or more nonzeros or terms (int32 indices)";

// Z = X Y (X: nx rows; Y: p columns, or Y = I with yrowptr null) or, with `transpose` (Y = I), Z = X' (p rows).  Z's pattern is
// allocated into `pat`, the pair lists into `lists`
int32_t sp_product(b200_ctx* ctx, int32_t nx, const int32_t* xrowptr, const int32_t* xcol, const int32_t* yrowptr, const int32_t* ycol, int32_t p, bool transpose,
                   std::vector<void*>& pat, std::vector<void*>& lists, DevCsr* z, PairLists* pl) {
  Scratch s;
  int64_t *cnt = nullptr, *off = nullptr;
  B200_TRY(dalloc(ctx, s.p, &cnt, (size_t)nx + 1));
  B200_TRY(dalloc(ctx, s.p, &off, (size_t)nx + 1));
  LAUNCH(ctx, sp_count_kernel, blocks((int64_t)nx + 1), AT, 0, nx, xrowptr, xcol, yrowptr, cnt);
  CHECK_LAUNCH(ctx);
  {
    size_t bytes = 0;
    CUDA_TRY(ctx, cub::DeviceScan::ExclusiveSum(nullptr, bytes, cnt, off, (int64_t)nx + 1, ctx->stream));
    void* tmp = nullptr;
    B200_TRY(dalloc(ctx, s.p, (char**)&tmp, bytes));
    CUDA_TRY(ctx, cub::DeviceScan::ExclusiveSum(tmp, bytes, cnt, off, (int64_t)nx + 1, ctx->stream));
  }
  int64_t nt64 = 0;
  CUDA_TRY(ctx, cudaMemcpyAsync(&nt64, off + nx, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (nt64 >= INT32_MAX) return ctx->fail(B200_ERR_UNSUPPORTED, AMG_PRODUCT_LIMIT, __FILE__, __LINE__);
  const int32_t nt = (int32_t)nt64;
  uint64_t *k0 = nullptr, *k1 = nullptr;
  int32_t *i0 = nullptr, *i1 = nullptr, *tx = nullptr, *ty = nullptr, *head = nullptr, *hs = nullptr;
  B200_TRY(dalloc(ctx, s.p, &k0, nt)); B200_TRY(dalloc(ctx, s.p, &k1, nt));
  B200_TRY(dalloc(ctx, s.p, &i0, nt)); B200_TRY(dalloc(ctx, s.p, &i1, nt));
  B200_TRY(dalloc(ctx, s.p, &tx, nt)); B200_TRY(dalloc(ctx, s.p, &ty, nt));
  const uint64_t kmax = (uint64_t)nx * (uint64_t)std::max(p, 1) - 1;   // the largest key
  int end_bit = 1;
  while (end_bit < 64 && (kmax >> end_bit) != 0) ++end_bit;
  LAUNCH(ctx, sp_expand_kernel, blocks(nx), AT, 0, nx, xrowptr, xcol, yrowptr, ycol, (uint64_t)p, (int)transpose, (const int64_t*)off, k0, i0, tx, ty);
  CHECK_LAUNCH(ctx);
  cub::DoubleBuffer<uint64_t> keys(k0, k1);
  cub::DoubleBuffer<int32_t> vals(i0, i1);
  {
    size_t bytes = 0;
    CUDA_TRY(ctx, cub::DeviceRadixSort::SortPairs(nullptr, bytes, keys, vals, nt, 0, end_bit, ctx->stream));
    void* tmp = nullptr;
    B200_TRY(dalloc(ctx, s.p, (char**)&tmp, bytes));
    CUDA_TRY(ctx, cub::DeviceRadixSort::SortPairs(tmp, bytes, keys, vals, nt, 0, end_bit, ctx->stream));
  }
  B200_TRY(dalloc(ctx, s.p, &head, (size_t)nt + 1));
  B200_TRY(dalloc(ctx, s.p, &hs, (size_t)nt + 1));
  LAUNCH(ctx, sp_heads_kernel, blocks((int64_t)nt + 1), AT, 0, nt, (const uint64_t*)keys.Current(), head);
  CHECK_LAUNCH(ctx);
  B200_TRY(scan_i32(ctx, head, hs, (int64_t)nt + 1));
  int32_t nout = 0;
  CUDA_TRY(ctx, cudaMemcpyAsync(&nout, hs + nt, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  z->nrows = transpose ? p : nx;
  z->nnz = nout;
  B200_TRY(dalloc(ctx, pat, &z->rowptr, (size_t)z->nrows + 1));
  B200_TRY(dalloc(ctx, pat, &z->col, nout));
  *pl = PairLists();
  B200_TRY(dalloc(ctx, lists, &pl->x, nt));
  if (!transpose) {
    B200_TRY(dalloc(ctx, lists, &pl->ptr, (size_t)nout + 1));
    B200_TRY(dalloc(ctx, lists, &pl->y, nt));
  }
  LAUNCH(ctx, sp_compress_kernel, blocks((int64_t)nt + 1), AT, 0, nt, z->nrows, transpose ? (uint64_t)nx : (uint64_t)p, (const uint64_t*)keys.Current(),
         (const int32_t*)vals.Current(), (const int32_t*)hs, (const int32_t*)tx, (const int32_t*)ty, z->rowptr, z->col, pl->ptr, pl->x, pl->y);
  CHECK_LAUNCH(ctx);
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return B200_OK;
}

void free_hierarchy(b200_amg* amg) {
  if (amg->gexec) { cudaStreamSynchronize(amg->ctx->stream); cudaGraphExecDestroy(amg->gexec); amg->gexec = nullptr; }
  cudaStreamSynchronize(amg->ctx->stream);
  for (void* p : amg->owned) cudaFree(p);
  amg->owned.clear();
  amg->lev.clear();
  amg->d_dense = amg->d_ainv = nullptr;
  amg->d_ipiv = nullptr;
  amg->built = amg->refreshed = 0;
  amg->graph_unavailable = false;
}

// the vectors of a level whose pattern (rowptr, col) is on the device; its diagonal positions
int32_t level_vectors(b200_amg* amg, AmgLevel& L) {
  b200_ctx* ctx = amg->ctx;
  auto& o = amg->owned;
  B200_TRY(dalloc(ctx, o, &L.diag, L.n));
  B200_TRY(dalloc(ctx, o, &L.val, L.nnz)); B200_TRY(dalloc(ctx, o, &L.dinv, L.n));
  B200_TRY(dalloc(ctx, o, &L.x, L.n)); B200_TRY(dalloc(ctx, o, &L.x2, L.n)); B200_TRY(dalloc(ctx, o, &L.b, L.n)); B200_TRY(dalloc(ctx, o, &L.r, L.n));
  LAUNCH(ctx, amg_diag_kernel, blocks(L.n), AT, 0, L.n, (const int32_t*)L.rowptr, (const int32_t*)L.col, L.diag);
  CHECK_LAUNCH(ctx);
  return B200_OK;
}

// level 0 from the caller's values, on a freed hierarchy
int32_t level0(b200_amg* amg, const double* nzval) {
  b200_ctx* ctx = amg->ctx;
  free_hierarchy(amg);
  const int32_t none = INT_MAX;
  CUDA_TRY(ctx, cudaMemcpyAsync(amg->d_info, &none, sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
  amg->lev.resize(1);
  AmgLevel& L = amg->lev[0];
  L.n = (int32_t)amg->n; L.nnz = (int32_t)amg->nnz;
  B200_TRY(upload(ctx, amg->owned, &L.rowptr, amg->rowptr0));
  B200_TRY(upload(ctx, amg->owned, &L.col, amg->col0));
  B200_TRY(level_vectors(amg, L));
  LAUNCH(ctx, amg_gather_kernel, blocks(L.nnz), AT, 0, L.nnz, (const int32_t*)amg->d_map0, nzval, L.val);
  CHECK_LAUNCH(ctx);
  return B200_OK;
}

// with P_l's pattern on the device: R = P' with its gather map, the pair lists of A P and R (A P), and level l + 1's pattern
int32_t galerkin_pattern(b200_amg* amg, int32_t l, int32_t nc) {
  b200_ctx* ctx = amg->ctx;
  auto& o = amg->owned;
  Scratch s;
  AmgLevel& L = amg->lev[l];
  DevCsr r, ap, c;
  PairLists lr, lap, lac;
  B200_TRY(sp_product(ctx, L.n, L.prowptr, L.pcol, nullptr, nullptr, nc, true, o, o, &r, &lr));
  L.rrowptr = r.rowptr; L.rcol = r.col; L.rmap = lr.x;
  B200_TRY(dalloc(ctx, o, &L.rval, L.pnnz));
  B200_TRY(sp_product(ctx, L.n, L.rowptr, L.col, L.prowptr, L.pcol, nc, false, s.p, o, &ap, &lap));
  L.apnnz = ap.nnz; L.ap_ptr = lap.ptr; L.ap_x = lap.x; L.ap_y = lap.y;
  B200_TRY(dalloc(ctx, o, &L.apval, L.apnnz));
  B200_TRY(sp_product(ctx, nc, L.rrowptr, L.rcol, ap.rowptr, ap.col, nc, false, o, o, &c, &lac));
  L.ac_ptr = lac.ptr; L.ac_x = lac.x; L.ac_y = lac.y;
  AmgLevel C;
  C.n = nc; C.nnz = c.nnz; C.rowptr = c.rowptr; C.col = c.col;
  amg->lev.push_back(C);   // L is not used past this point
  B200_TRY(level_vectors(amg, amg->lev.back()));
  return B200_OK;
}

// every value of level l's P, R and of A_{l+1} from A_l's values (refresh and rebuild alike)
int32_t level_values(b200_amg* amg, int32_t l) {
  b200_ctx* ctx = amg->ctx;
  AmgLevel &L = amg->lev[l], &Cl = amg->lev[l + 1];
  LAUNCH(ctx, amg_dinv_kernel, blocks(L.n), AT, 0, L.n, (const int32_t*)L.diag, (const double*)L.val, L.dinv, l, amg->d_info);
  if (amg->method == AMG_SA) {
    CUDA_TRY(ctx, cudaMemsetAsync(L.rho, 0, sizeof(unsigned long long), ctx->stream));
    LAUNCH(ctx, sa_rho_kernel, blocks(L.n), AT, 0, L.n, (const int32_t*)L.rowptr, (const int32_t*)L.diag, (const double*)L.val, L.rho);
    LAUNCH(ctx, amg_pair_product_kernel, blocks(L.pnnz), AT, 0, L.pnnz, (const int32_t*)L.at_ptr, (const int32_t*)L.at_x, (const int32_t*)L.at_y,
           (const double*)L.val, (const double*)L.tval, L.atval);
    LAUNCH(ctx, sa_p_kernel, blocks(L.n), AT, 0, L.n, (const int32_t*)L.prowptr, (const int32_t*)L.pcol, (const int32_t*)L.trowptr, (const int32_t*)L.tcol,
           (const double*)L.tval, (const double*)L.dinv, (const double*)L.atval, (const unsigned long long*)L.rho, amg->smooth_omega, L.pval);
  } else {
    LAUNCH(ctx, amg_interp_kernel, blocks(L.n), AT, 0, L.n, (const int32_t*)L.rowptr, (const int32_t*)L.col, (const int32_t*)L.diag, (const double*)L.val,
           (const int32_t*)L.prowptr, (const int32_t*)L.pmap, L.pval, l, amg->d_info);
  }
  LAUNCH(ctx, amg_gather_kernel, blocks(L.pnnz), AT, 0, L.pnnz, (const int32_t*)L.rmap, (const double*)L.pval, L.rval);
  LAUNCH(ctx, amg_pair_product_kernel, blocks(L.apnnz), AT, 0, L.apnnz, (const int32_t*)L.ap_ptr, (const int32_t*)L.ap_x, (const int32_t*)L.ap_y,
         (const double*)L.val, (const double*)L.pval, L.apval);
  LAUNCH(ctx, amg_pair_product_kernel, blocks(Cl.nnz), AT, 0, Cl.nnz, (const int32_t*)L.ac_ptr, (const int32_t*)L.ac_x, (const int32_t*)L.ac_y,
         (const double*)L.rval, (const double*)L.apval, Cl.val);
  CHECK_LAUNCH(ctx);
  return B200_OK;
}

// the Ruge-Stueben rebuild: strength and the splitting on the host, every pattern and value on the device
int32_t rebuild_rs(b200_amg* amg, const double* nzval) {
  b200_ctx* ctx = amg->ctx;
  const b200_amg_opts& o = amg->o;
  HostLevel h;
  h.n = (int32_t)amg->n; h.rowptr = amg->rowptr0; h.col = amg->col0;
  {
    std::vector<double> nz;
    B200_TRY(download(ctx, nz, nzval, amg->nnz));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    h.val.resize(amg->nnz);
    for (int64_t q = 0; q < amg->nnz; ++q) h.val[q] = nz[amg->map0[q]];
  }
  B200_TRY(level0(amg, nzval));
  for (;;) {
    const int32_t l = (int32_t)amg->lev.size() - 1;
    if (h.n <= o.max_coarse || l + 1 >= o.max_levels) break;
    std::vector<char> strong;
    std::vector<int32_t> cf, prowptr, pcol, pmap;
    strength(h.n, h.rowptr, h.col, h.val.data(), o.theta, strong);
    const int64_t nc = rs_split(h.n, h.rowptr, h.col, strong, cf);
    if (nc == 0 || nc == h.n) { amg->stall = nc == 0 ? AMG_STOP_NONE : AMG_STOP_ALL; break; }
    interpolation_pattern(h, strong, cf, prowptr, pcol, pmap);
    AmgLevel& L = amg->lev[l];
    L.pnnz = prowptr[h.n];
    B200_TRY(upload(ctx, amg->owned, &L.prowptr, prowptr));
    B200_TRY(upload(ctx, amg->owned, &L.pcol, pcol));
    B200_TRY(upload(ctx, amg->owned, &L.pmap, pmap));
    B200_TRY(dalloc(ctx, amg->owned, &L.pval, L.pnnz));
    B200_TRY(galerkin_pattern(amg, l, (int32_t)nc));
    B200_TRY(level_values(amg, l));
    const AmgLevel& C = amg->lev[l + 1];
    h.n = C.n;
    B200_TRY(download(ctx, h.rowptr, C.rowptr, (size_t)C.n + 1));
    B200_TRY(download(ctx, h.col, C.col, C.nnz));
    B200_TRY(download(ctx, h.val, C.val, C.nnz));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  }
  return B200_OK;
}

// the smoothed-aggregation rebuild, every step on the device; the host reads back sizes only
int32_t rebuild_sa(b200_amg* amg, const double* nzval) {
  b200_ctx* ctx = amg->ctx;
  const b200_amg_opts& o = amg->o;
  auto& own = amg->owned;
  B200_TRY(level0(amg, nzval));
  Scratch cand;   // the candidate b of every level so far (ones on level 0)
  double* b = nullptr;
  {
    std::vector<double> ones(amg->n, 1.0);
    B200_TRY(upload(ctx, cand.p, &b, ones));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  }
  for (;;) {
    const int32_t l = (int32_t)amg->lev.size() - 1;
    AmgLevel& L = amg->lev[l];
    const int32_t n = L.n;
    if (n <= o.max_coarse || l + 1 >= o.max_levels) break;
    Scratch s;
    DevCsr at;
    PairLists lat;
    B200_TRY(sp_product(ctx, n, L.rowptr, L.col, nullptr, nullptr, n, true, s.p, s.p, &at, &lat));   // A' for the symmetric graph
    uint8_t* strong = nullptr;
    B200_TRY(dalloc(ctx, s.p, &strong, L.nnz));
    LAUNCH(ctx, sa_strength_kernel, blocks(n), AT, 0, n, (const int32_t*)L.rowptr, (const int32_t*)L.col, (const int32_t*)L.diag, (const double*)L.val, o.theta, strong);
    const SaGraph g{L.rowptr, L.col, at.rowptr, at.col, lat.x, strong};
    // distance-2 maximal independent set
    uint64_t *key = nullptr, *m1 = nullptr, *m2 = nullptr;
    int32_t* und = nullptr;
    B200_TRY(dalloc(ctx, s.p, &key, n)); B200_TRY(dalloc(ctx, s.p, &m1, n)); B200_TRY(dalloc(ctx, s.p, &m2, n));
    B200_TRY(dalloc(ctx, s.p, &und, 1));
    LAUNCH(ctx, sa_mis_init_kernel, blocks(n), AT, 0, n, g, key);
    for (int32_t left = 1; left > 0;) {
      CUDA_TRY(ctx, cudaMemsetAsync(und, 0, sizeof(int32_t), ctx->stream));
      LAUNCH(ctx, sa_max_kernel, blocks(n), AT, 0, n, g, (const uint64_t*)key, m1);
      LAUNCH(ctx, sa_max_kernel, blocks(n), AT, 0, n, g, (const uint64_t*)m1, m2);
      LAUNCH(ctx, sa_mis_update_kernel, blocks(n), AT, 0, n, key, (const uint64_t*)m2, und);
      CHECK_LAUNCH(ctx);
      CUDA_TRY(ctx, cudaMemcpyAsync(&left, und, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
      CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    }
    // aggregates: roots numbered in index order, then two passes
    int32_t *flag = nullptr, *rid = nullptr, *agg1 = nullptr, *agg2 = nullptr;
    B200_TRY(dalloc(ctx, s.p, &flag, (size_t)n + 1)); B200_TRY(dalloc(ctx, s.p, &rid, (size_t)n + 1));
    B200_TRY(dalloc(ctx, s.p, &agg1, n)); B200_TRY(dalloc(ctx, s.p, &agg2, n));
    LAUNCH(ctx, sa_root_flag_kernel, blocks((int64_t)n + 1), AT, 0, n, (const uint64_t*)key, flag);
    CHECK_LAUNCH(ctx);
    B200_TRY(scan_i32(ctx, flag, rid, (int64_t)n + 1));
    int32_t na = 0;
    CUDA_TRY(ctx, cudaMemcpyAsync(&na, rid + n, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    if (na == 0 || na == n) { amg->stall = na == 0 ? AMG_STOP_NONE : AMG_STOP_ALL; break; }
    LAUNCH(ctx, sa_pass1_kernel, blocks(n), AT, 0, n, g, (const uint64_t*)key, (const int32_t*)rid, agg1);
    LAUNCH(ctx, sa_pass2_kernel, blocks(n), AT, 0, n, g, (const int32_t*)agg1, agg2);
    // T: one entry per aggregated row, b / ||b on the aggregate||; the next level's b is the aggregates' norms
    LAUNCH(ctx, sa_tflag_kernel, blocks((int64_t)n + 1), AT, 0, n, (const int32_t*)agg2, flag);
    CHECK_LAUNCH(ctx);
    B200_TRY(dalloc(ctx, own, &L.trowptr, (size_t)n + 1));
    B200_TRY(scan_i32(ctx, flag, L.trowptr, (int64_t)n + 1));
    CUDA_TRY(ctx, cudaMemcpyAsync(&L.tnnz, L.trowptr + n, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    B200_TRY(dalloc(ctx, own, &L.tcol, L.tnnz));
    B200_TRY(dalloc(ctx, own, &L.tval, L.tnnz));
    LAUNCH(ctx, sa_tcol_kernel, blocks(n), AT, 0, n, (const int32_t*)agg2, (const int32_t*)L.trowptr, L.tcol);
    CHECK_LAUNCH(ctx);
    DevCsr mem;
    PairLists lmem;
    B200_TRY(sp_product(ctx, n, L.trowptr, L.tcol, nullptr, nullptr, na, true, s.p, s.p, &mem, &lmem));
    double* nrm = nullptr;
    B200_TRY(dalloc(ctx, cand.p, &nrm, na));
    LAUNCH(ctx, sa_norm_kernel, blocks(na), AT, 0, na, (const int32_t*)mem.rowptr, (const int32_t*)mem.col, (const double*)b, nrm);
    LAUNCH(ctx, sa_tval_kernel, blocks(n), AT, 0, n, (const int32_t*)L.trowptr, (const int32_t*)L.tcol, (const double*)b, (const double*)nrm, L.tval);
    CHECK_LAUNCH(ctx);
    b = nrm;
    // P on A T's pattern, with A T's pair lists
    DevCsr pz;
    PairLists lpt;
    B200_TRY(sp_product(ctx, n, L.rowptr, L.col, L.trowptr, L.tcol, na, false, own, own, &pz, &lpt));
    L.pnnz = pz.nnz; L.prowptr = pz.rowptr; L.pcol = pz.col;
    L.at_ptr = lpt.ptr; L.at_x = lpt.x; L.at_y = lpt.y;
    B200_TRY(dalloc(ctx, own, &L.pval, L.pnnz));
    B200_TRY(dalloc(ctx, own, &L.atval, L.pnnz));
    B200_TRY(dalloc(ctx, own, &L.rho, 1));
    B200_TRY(galerkin_pattern(amg, l, na));
    B200_TRY(level_values(amg, l));
  }
  return B200_OK;
}

// either rebuild, then the coarsest level's workspace
int32_t rebuild(b200_amg* amg, const double* nzval) {
  b200_ctx* ctx = amg->ctx;
  amg->stall = AMG_STOP_SIZE;
  const int32_t rc = amg->method == AMG_SA ? rebuild_sa(amg, nzval) : rebuild_rs(amg, nzval);
  if (rc != B200_OK) { free_hierarchy(amg); return rc; }
  const int64_t nco = amg->lev.back().n;
  if (nco > AMG_DENSE_CAP) {
    // the advice names the cause: raising max_levels helps only when max_levels stopped the coarsening
    char msg[320];
    const int nlev = (int)amg->lev.size();
    if (amg->stall != AMG_STOP_SIZE) {
      const char* why = amg->method == AMG_SA ? (amg->stall == AMG_STOP_NONE ? "no aggregate: no node has a strong connection" : "every node is an aggregate root")
                                              : (amg->stall == AMG_STOP_NONE ? "no C point: no point has a strong connection" : "every point is a C point");
      snprintf(msg, sizeof(msg), "amg_setup: coarsening stalls at level %d of %lld unknowns (%s), above the %lld of the coarsest level's dense inverse",
               nlev, (long long)nco, why, (long long)AMG_DENSE_CAP);
    } else if (nco <= amg->o.max_coarse) {
      snprintf(msg, sizeof(msg), "amg_setup: the hierarchy ends at %lld unknowns (%d levels) by max_coarse = %d, above the %lld of the coarsest level's dense inverse: lower max_coarse",
               (long long)nco, nlev, (int)amg->o.max_coarse, (long long)AMG_DENSE_CAP);
    } else {
      snprintf(msg, sizeof(msg), "amg_setup: the hierarchy ends at %lld unknowns (%d levels), above the %lld of the coarsest level's dense inverse: raise max_levels",
               (long long)nco, nlev, (long long)AMG_DENSE_CAP);
    }
    free_hierarchy(amg);
    return ctx->fail(B200_ERR_UNSUPPORTED, msg, __FILE__, __LINE__);
  }
  int32_t st = dalloc(ctx, amg->owned, &amg->d_dense, (size_t)nco * nco);
  if (st == B200_OK) st = dalloc(ctx, amg->owned, &amg->d_ainv, (size_t)nco * nco);
  if (st == B200_OK) st = dalloc(ctx, amg->owned, &amg->d_ipiv, (size_t)nco);
  if (st == B200_OK && cudaStreamSynchronize(ctx->stream) != cudaSuccess) st = ctx->fail(B200_ERR_CUDA, "AMG: the rebuild failed on the device", __FILE__, __LINE__);
  if (st != B200_OK) { free_hierarchy(amg); return st; }
  amg->built = 1;
  return B200_OK;
}

// every value of the frozen hierarchy from the level-0 values; *info as b200_amg_setup reports it
int32_t refresh(b200_amg* amg, const double* nzval, int32_t* info) {
  b200_ctx* ctx = amg->ctx;
  const int32_t none = INT_MAX;
  CUDA_TRY(ctx, cudaMemcpyAsync(amg->d_info, &none, sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
  AmgLevel& L0 = amg->lev[0];
  LAUNCH(ctx, amg_gather_kernel, blocks(L0.nnz), AT, 0, L0.nnz, (const int32_t*)amg->d_map0, nzval, L0.val);
  const int32_t nlev = (int32_t)amg->lev.size();
  for (int32_t l = 0; l + 1 < nlev; ++l) B200_TRY(level_values(amg, l));
  CHECK_LAUNCH(ctx);
  int32_t h = 0;
  CUDA_TRY(ctx, cudaMemcpyAsync(&h, amg->d_info, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  *info = h == INT_MAX ? 0 : h;
  if (*info != 0) return B200_OK;  // no dense LU of values that are already not finite
  // the coarsest level: A_c = L U by getrf, then A_c^-1 = getrs(L U, I)
  AmgLevel& Lc = amg->lev[nlev - 1];
  const int64_t nc = Lc.n;
  CUDA_TRY(ctx, cudaMemsetAsync(amg->d_dense, 0, sizeof(double) * nc * nc, ctx->stream));
  LAUNCH(ctx, amg_densify_kernel, blocks(nc), AT, 0, (int32_t)nc, (const int32_t*)Lc.rowptr, (const int32_t*)Lc.col, (const double*)Lc.val, amg->d_dense);
  CHECK_LAUNCH(ctx);
  int32_t lu = 0;
  B200_TRY(b200_getrf(ctx, nc, amg->d_dense, nc, amg->d_ipiv, &lu));
  if (lu != 0) { *info = nlev; return B200_OK; }
  LAUNCH(ctx, amg_identity_kernel, blocks(nc * nc), AT, 0, nc, amg->d_ainv);
  CHECK_LAUNCH(ctx);
  B200_TRY(b200_getrs(ctx, nc, nc, amg->d_dense, nc, amg->d_ipiv, amg->d_ainv, nc));
  return B200_OK;
}

// one V-cycle below level l for the right-hand side b; *xout = the level's result buffer
int32_t vcycle(b200_amg* amg, int32_t l, const double* b, double** xout) {
  b200_ctx* ctx = amg->ctx;
  const b200_amg_opts& o = amg->o;
  AmgLevel& L = amg->lev[l];
  if (l + 1 == (int32_t)amg->lev.size()) {
    B200_TRY(b200_gemv(ctx, 0, L.n, L.n, amg->d_ainv, L.n, b, L.x));
    *xout = L.x;
    return B200_OK;
  }
  double *x = L.x, *y = L.x2;
  const int g = blocks(L.n);
  if (o.presweeps == 0) {
    CUDA_TRY(ctx, cudaMemsetAsync(x, 0, sizeof(double) * L.n, ctx->stream));
  } else {
    LAUNCH(ctx, amg_jacobi0_kernel, g, AT, 0, L.n, o.omega, (const double*)L.dinv, b, x);
    for (int s = 1; s < o.presweeps; ++s) {
      LAUNCH(ctx, amg_residual_kernel, g, AT, 0, L.n, (const int32_t*)L.rowptr, (const int32_t*)L.col, (const double*)L.val, (const double*)x, b, 1, o.omega,
             (const double*)L.dinv, y);
      std::swap(x, y);
    }
  }
  LAUNCH(ctx, amg_residual_kernel, g, AT, 0, L.n, (const int32_t*)L.rowptr, (const int32_t*)L.col, (const double*)L.val, (const double*)x, b, 0, o.omega,
         (const double*)L.dinv, L.r);
  AmgLevel& Cl = amg->lev[l + 1];
  LAUNCH(ctx, amg_spmv_kernel, blocks(Cl.n), AT, 0, Cl.n, (const int32_t*)L.rrowptr, (const int32_t*)L.rcol, (const double*)L.rval, (const double*)L.r, 0, Cl.b);
  double* xc = nullptr;
  B200_TRY(vcycle(amg, l + 1, Cl.b, &xc));
  LAUNCH(ctx, amg_spmv_kernel, g, AT, 0, L.n, (const int32_t*)L.prowptr, (const int32_t*)L.pcol, (const double*)L.pval, (const double*)xc, 1, x);
  for (int s = 0; s < o.postsweeps; ++s) {
    LAUNCH(ctx, amg_residual_kernel, g, AT, 0, L.n, (const int32_t*)L.rowptr, (const int32_t*)L.col, (const double*)L.val, (const double*)x, b, 1, o.omega,
           (const double*)L.dinv, y);
    std::swap(x, y);
  }
  CHECK_LAUNCH(ctx);
  *xout = x;
  return B200_OK;
}
// the handle of either method: the level-0 CSR view of the caller's CSC pattern and its gather map
int32_t create(b200_ctx* ctx, const char* who, int64_t n, const int64_t* colptr, const int64_t* rowval, int32_t base, const b200_amg_opts& o, int method,
               double smooth_omega, b200_amg** out) {
  const std::string w(who);
  B200_REQUIRE(ctx, n > 0 && colptr && rowval && out && (base == 0 || base == 1), (w + ": bad arguments").c_str());
  const int64_t nnz = colptr[n] - colptr[0];
  B200_REQUIRE(ctx, colptr[0] == base && nnz >= 0, (w + ": colptr must start at the index base").c_str());
  B200_REQUIRE(ctx, n < INT32_MAX && nnz < INT32_MAX, (w + ": n and nnz must be below 2^31 (int32 CSR indices)").c_str());
  std::vector<int32_t> rowptr, col, map, diag;
  const std::string err = b200i_csr_of_csc(who, n, colptr, rowval, base, true, rowptr, col, map, diag);
  if (!err.empty()) return ctx->fail(B200_ERR_INVALID, err.c_str(), __FILE__, __LINE__);
  b200_amg* amg = new b200_amg();
  amg->ctx = ctx; amg->n = n; amg->nnz = nnz; amg->o = o; amg->method = method; amg->smooth_omega = smooth_omega;
  amg->rowptr0 = std::move(rowptr); amg->col0 = std::move(col); amg->map0 = std::move(map);
  bool ok = cudaMalloc(&amg->d_map0, sizeof(int32_t) * std::max<int64_t>(nnz, 1)) == cudaSuccess && cudaMalloc(&amg->d_info, sizeof(int32_t)) == cudaSuccess &&
            (nnz == 0 || cudaMemcpyAsync(amg->d_map0, amg->map0.data(), sizeof(int32_t) * nnz, cudaMemcpyHostToDevice, ctx->stream) == cudaSuccess) &&
            cudaStreamSynchronize(ctx->stream) == cudaSuccess;
  if (!ok) { cudaGetLastError(); b200_amg_destroy(amg); return ctx->fail(B200_ERR_NOMEM, "AMG: out of device memory", __FILE__, __LINE__); }
  *out = amg;
  return B200_OK;
}
}  // namespace

extern "C" {
void b200_amg_opts_default(b200_amg_opts* o) {
  o->theta = 0.25;
  o->omega = 2.0 / 3.0;
  o->presweeps = 1;
  o->postsweeps = 1;
  o->max_levels = 10;
  o->max_coarse = 10;
}

void b200_sa_opts_default(b200_sa_opts* o) {
  o->theta = 0.08;
  o->omega = 2.0 / 3.0;
  o->presweeps = 1;
  o->postsweeps = 1;
  o->max_levels = 10;
  o->max_coarse = 10;
  o->smooth_omega = 4.0 / 3.0;
}

int32_t b200_amg_destroy(b200_amg* amg) {
  if (!amg) return B200_OK;
  B200_DEVICE_GUARD(amg->ctx);
  free_hierarchy(amg);
  cudaFree(amg->d_map0); cudaFree(amg->d_info);
  delete amg;
  return B200_OK;
}

int32_t b200_amg_create(b200_ctx* ctx, int64_t n, const int64_t* colptr, const int64_t* rowval, int32_t base, const b200_amg_opts* opts, b200_amg** out) {
  B200_DEVICE_GUARD(ctx);
  b200_amg_opts o;
  b200_amg_opts_default(&o);
  if (opts) o = *opts;
  B200_REQUIRE(ctx, o.theta >= 0.0 && o.theta <= 1.0 && o.omega > 0.0 && o.presweeps >= 0 && o.postsweeps >= 0 && o.max_levels >= 1 && o.max_coarse >= 1,
               "amg_create: options out of range (0 <= theta <= 1, omega > 0, sweeps >= 0, max_levels >= 1, max_coarse >= 1)");
  return create(ctx, "amg_create", n, colptr, rowval, base, o, AMG_RS, 0.0, out);
}

int32_t b200_amg_create_sa(b200_ctx* ctx, int64_t n, const int64_t* colptr, const int64_t* rowval, int32_t base, const b200_sa_opts* opts, b200_amg** out) {
  B200_DEVICE_GUARD(ctx);
  b200_sa_opts s;
  b200_sa_opts_default(&s);
  if (opts) s = *opts;
  B200_REQUIRE(ctx, s.theta >= 0.0 && s.theta <= 1.0 && s.omega > 0.0 && s.presweeps >= 0 && s.postsweeps >= 0 && s.max_levels >= 1 && s.max_coarse >= 1 &&
                        s.smooth_omega > 0.0 && std::isfinite(s.omega) && std::isfinite(s.smooth_omega),
               "amg_create_sa: options out of range (0 <= theta <= 1, omega > 0, sweeps >= 0, max_levels >= 1, max_coarse >= 1, smooth_omega > 0)");
  b200_amg_opts o;
  o.theta = s.theta; o.omega = s.omega; o.presweeps = s.presweeps; o.postsweeps = s.postsweeps; o.max_levels = s.max_levels; o.max_coarse = s.max_coarse;
  return create(ctx, "amg_create_sa", n, colptr, rowval, base, o, AMG_SA, s.smooth_omega, out);
}

int32_t b200_amg_setup(b200_amg* amg, const double* nzval, int32_t rebuild_flag, int32_t* info_host) {
  B200_DEVICE_GUARD(amg ? amg->ctx : nullptr);
  b200_ctx* ctx = amg->ctx;
  B200_REQUIRE(ctx, nzval, "amg_setup: bad arguments");
  B200_REQUIRE(ctx, rebuild_flag || amg->built, "amg_setup: a refresh (rebuild = 0) needs a hierarchy: rebuild first");
  if (rebuild_flag) B200_TRY(rebuild(amg, nzval));
  int32_t info = 0;
  amg->refreshed = 0;
  B200_TRY(refresh(amg, nzval, &info));
  amg->refreshed = 1;
  if (info_host) *info_host = info;
  return B200_OK;
}

int32_t b200_amg_solve(b200_amg* amg, const double* b, double* x) {
  B200_DEVICE_GUARD(amg ? amg->ctx : nullptr);
  b200_ctx* ctx = amg->ctx;
  B200_REQUIRE(ctx, amg->refreshed, "amg_solve before amg_setup");
  const size_t bytes = sizeof(double) * amg->n;
  AmgLevel& L0 = amg->lev[0];
  if (!amg->gexec && !amg->graph_unavailable && !ctx->prof_on) {
    cudaGraph_t graph = nullptr;
    const int64_t l0 = ctx->launches;
    double* res = nullptr;
    if (cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
      const int32_t rc = vcycle(amg, 0, L0.b, &res);
      const cudaError_t e = cudaStreamEndCapture(ctx->stream, &graph);
      if (rc == B200_OK && e == cudaSuccess && graph && cudaGraphInstantiate(&amg->gexec, graph, 0) == cudaSuccess) {
        amg->gres = res;
        amg->glaunches = ctx->launches - l0;
      } else {
        amg->gexec = nullptr;
        amg->graph_unavailable = true;
        cudaGetLastError();
      }
      if (graph) cudaGraphDestroy(graph);
      ctx->launches = l0;  // nothing ran yet
    } else {
      amg->graph_unavailable = true;
      cudaGetLastError();
    }
  }
  if (amg->gexec) {
    CUDA_TRY(ctx, cudaMemcpyAsync(L0.b, b, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
    CUDA_TRY(ctx, cudaGraphLaunch(amg->gexec, ctx->stream));
    ctx->launches += amg->glaunches;
    CUDA_TRY(ctx, cudaMemcpyAsync(x, amg->gres, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
    return B200_OK;
  }
  CUDA_TRY(ctx, cudaMemcpyAsync(L0.b, b, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
  double* res = nullptr;
  B200_TRY(vcycle(amg, 0, L0.b, &res));
  CUDA_TRY(ctx, cudaMemcpyAsync(x, res, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
  return B200_OK;
}

int32_t b200_amg_levels(b200_amg* amg, int32_t* nlev, int64_t* nper, int64_t* nnzper, int32_t cap) {
  B200_REQUIRE(amg->ctx, amg->built && nlev, "amg_levels before the first rebuild, or bad arguments");
  *nlev = (int32_t)amg->lev.size();
  for (int32_t l = 0; l < *nlev && l < cap; ++l) {
    if (nper) nper[l] = amg->lev[l].n;
    if (nnzper) nnzper[l] = amg->lev[l].nnz;
  }
  return B200_OK;
}

int32_t b200_amg_export(b200_amg* amg, int32_t level, int32_t what, int32_t* rowptr, int32_t* col, double* val) {
  B200_DEVICE_GUARD(amg ? amg->ctx : nullptr);
  b200_ctx* ctx = amg->ctx;
  const int32_t nlev = (int32_t)amg->lev.size();
  B200_REQUIRE(ctx, amg->refreshed && rowptr && level >= 0 && level < nlev &&
                        (what == B200_AMG_EXPORT_A || ((what == B200_AMG_EXPORT_P || (what == B200_AMG_EXPORT_T && amg->method == AMG_SA)) && level + 1 < nlev)),
               "amg_export: bad arguments (P and T exist on every level but the coarsest, T on smoothed-aggregation handles only), or no setup yet");
  const AmgLevel& L = amg->lev[level];
  const int32_t* rp = what == B200_AMG_EXPORT_A ? L.rowptr : what == B200_AMG_EXPORT_P ? L.prowptr : L.trowptr;
  const int32_t* cl = what == B200_AMG_EXPORT_A ? L.col : what == B200_AMG_EXPORT_P ? L.pcol : L.tcol;
  const double* vl = what == B200_AMG_EXPORT_A ? L.val : what == B200_AMG_EXPORT_P ? L.pval : L.tval;
  const int32_t nz = what == B200_AMG_EXPORT_A ? L.nnz : what == B200_AMG_EXPORT_P ? L.pnnz : L.tnnz;
  CUDA_TRY(ctx, cudaMemcpyAsync(rowptr, rp, sizeof(int32_t) * (L.n + 1), cudaMemcpyDeviceToHost, ctx->stream));
  if (col) CUDA_TRY(ctx, cudaMemcpyAsync(col, cl, sizeof(int32_t) * nz, cudaMemcpyDeviceToHost, ctx->stream));
  if (val) CUDA_TRY(ctx, cudaMemcpyAsync(val, vl, sizeof(double) * nz, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return B200_OK;
}

int32_t b200_amg_linop(b200_amg* amg, b200_linop** out) {
  B200_DEVICE_GUARD(amg ? amg->ctx : nullptr);
  B200_REQUIRE(amg->ctx, out, "amg_linop: bad arguments");
  b200_linop* op = new b200_linop();
  memset(op, 0, sizeof(*op));
  op->ctx = amg->ctx; op->kind = LINOP_AMG; op->n = amg->n; op->amg = amg;
  *out = op;
  return B200_OK;
}

int32_t b200_amg_split(int64_t n, const int64_t* colptr, const int64_t* rowval, const double* nzval, int32_t base, double theta, int32_t* cf_out,
                       int64_t* ncoarse) {
  if (n <= 0 || n >= INT32_MAX || !colptr || !rowval || !nzval || !cf_out || (base != 0 && base != 1) || colptr[0] != base ||
      colptr[n] - colptr[0] >= INT32_MAX || !(theta >= 0.0 && theta <= 1.0))
    return B200_ERR_INVALID;
  std::vector<int32_t> rowptr, col, map, diag;
  if (!b200i_csr_of_csc("amg_split", n, colptr, rowval, base, false, rowptr, col, map, diag).empty()) return B200_ERR_INVALID;
  std::vector<double> val(map.size());
  for (size_t q = 0; q < map.size(); ++q) val[q] = nzval[map[q]];
  std::vector<char> strong;
  std::vector<int32_t> cf;
  strength((int32_t)n, rowptr, col, val.data(), theta, strong);
  const int64_t nc = rs_split((int32_t)n, rowptr, col, strong, cf);
  std::copy(cf.begin(), cf.end(), cf_out);
  if (ncoarse) *ncoarse = nc;
  return B200_OK;
}
}  // extern "C"
