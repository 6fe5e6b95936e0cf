// amg.cu — classical Ruge-Stueben algebraic multigrid of an assembled sparse matrix, the second preconditioner of GMRES on the
// sparse route (`KrylovJL_GMRES(precs = ...)` with `aspreconditioner(ruge_stuben(W))` and Jacobi smoothing,
// docs/src/tutorials/large_systems.md:244-316).  DESIGN.md §4h states the rules; in short:
//
//   * strength: j strongly influences i (j != i) when |a_ij| >= theta max_{k != i} |a_ik| and a_ij != 0;
//   * splitting: the Ruge-Stueben first pass, points with no strong connection in either direction F, then repeatedly the
//     unassigned point of largest lambda (ties: smallest index) becomes C, the unassigned points it influences F, and every
//     unassigned point influencing a new F point gains one in lambda; no second pass;
//   * direct interpolation from the strong C-neighbours, sign-split (alpha for negative, beta for positive entries);
//   * Galerkin coarse operators A_{l+1} = R A_l P with R = P' stored explicitly; the coarsest level's explicit inverse.
//
// Where the work runs:
//   * rebuild (host, once per pattern): the values come down once; strength, splitting, the patterns of P, R, A P and of every
//     coarse operator, and the product index lists are built level by level (the host computes values only to choose the next
//     splitting).  Then the patterns go up and the device refresh computes every value;
//   * refresh (device, every later fresh Jacobian): gather, interpolation weights (one thread per row), R = P' by a gather,
//     A P and R (A P) by one pair-list product kernel, inverse diagonals, the coarsest inverse by getrf / getrs.  Every sum runs
//     in a fixed order and there is no floating-point atomic: a refresh is bit-reproducible, and a rebuild gives the same bits;
//   * apply: one V-cycle, damped Jacobi (the first pre-sweep from x = 0 is x = omega D^-1 b), residual, restriction, prolongation
//     and the coarsest GEMV, captured once per rebuild into a CUDA graph (a refresh writes values in place, so the graph stays valid).
#include "common.cuh"
#include <algorithm>
#include <climits>
#include <cmath>
#include <queue>
#include <vector>

namespace {
constexpr int AT = 256;
constexpr int64_t AMG_DENSE_CAP = 4096;  // largest coarsest level that gets an explicit dense inverse

// one level of the hierarchy on the device; P, R and the product lists exist on every level but the coarsest
struct AmgLevel {
  int32_t n = 0, nnz = 0;                    // A_l
  int32_t *rowptr = nullptr, *col = nullptr, *diag = nullptr;
  double *val = nullptr, *dinv = nullptr;
  int32_t pnnz = 0;                          // P_l: n x n_{l+1}
  int32_t *prowptr = nullptr, *pcol = nullptr, *pmap = nullptr;  // pmap: P position -> A_l position (-1 on C rows)
  double* pval = nullptr;
  int32_t *rrowptr = nullptr, *rcol = nullptr, *rmap = nullptr;  // R = P': rmap = R position -> P position
  double* rval = nullptr;
  int32_t apnnz = 0;                         // A_l P_l: values only (the pair lists address them)
  double* apval = nullptr;
  int32_t *ap_ptr = nullptr, *ap_x = nullptr, *ap_y = nullptr;   // AP[q] = sum_t A[ap_x[t]] P[ap_y[t]], t in [ap_ptr[q], ap_ptr[q+1])
  int32_t *ac_ptr = nullptr, *ac_x = nullptr, *ac_y = nullptr;   // A_{l+1}[q] = sum_t R[ac_x[t]] AP[ac_y[t]]
  double *x = nullptr, *x2 = nullptr, *b = nullptr, *r = nullptr;
};

// host CSR of one level while the hierarchy is built
struct HostLevel {
  int32_t n = 0;
  std::vector<int32_t> rowptr, col, diag;
  std::vector<double> val;
  std::vector<int32_t> prowptr, pcol, pmap, rrowptr, rcol, rmap;
  std::vector<double> pval;
  std::vector<int32_t> ap_rowptr, ap_col, ap_ptr, ap_x, ap_y, ac_ptr, ac_x, ac_y;
};
}  // namespace

struct b200_amg {
  b200_ctx* ctx;
  int64_t n, nnz;
  b200_amg_opts o;
  std::vector<int32_t> rowptr0, col0, map0;  // level-0 CSR view of the caller's CSC pattern
  int32_t* d_map0 = nullptr;
  std::vector<AmgLevel> lev;
  std::vector<void*> owned;                  // device allocations of the current hierarchy
  double *d_dense = nullptr, *d_ainv = nullptr;  // coarsest level: LU workspace, explicit inverse
  int64_t* d_ipiv = nullptr;
  int32_t* d_info = nullptr;
  int built = 0, refreshed = 0;
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

inline int blocks(int64_t n) { return (int)std::max<int64_t>(1, (n + AT - 1) / AT); }

// ---------------------------------------------------------------- host: strength, splitting, interpolation, products
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

// out-pattern and pair list of the product X Y (CSR X: xrowptr/xcol, CSR Y: yrowptr/ycol); pairs address X and Y positions,
// in ascending X position within each output entry
void pair_product(int32_t n, const std::vector<int32_t>& xrowptr, const std::vector<int32_t>& xcol, const std::vector<int32_t>& yrowptr,
                  const std::vector<int32_t>& ycol, std::vector<int32_t>& orowptr, std::vector<int32_t>& ocol, std::vector<int32_t>& ptr,
                  std::vector<int32_t>& px, std::vector<int32_t>& py, const char** err) {
  orowptr.assign(n + 1, 0);
  ocol.clear(); ptr.assign(1, 0); px.clear(); py.clear();
  struct Trip { int32_t c, x, y; };
  std::vector<Trip> row;
  for (int32_t i = 0; i < n; ++i) {
    row.clear();
    for (int32_t q = xrowptr[i]; q < xrowptr[i + 1]; ++q)
      for (int32_t t = yrowptr[xcol[q]]; t < yrowptr[xcol[q] + 1]; ++t) row.push_back({ycol[t], q, t});
    std::stable_sort(row.begin(), row.end(), [](const Trip& a, const Trip& b) { return a.c < b.c; });
    for (size_t k = 0; k < row.size(); ++k) {
      if (k == 0 || row[k].c != row[k - 1].c) {
        if (k > 0) ptr.push_back((int32_t)px.size());
        ocol.push_back(row[k].c);
      }
      px.push_back(row[k].x); py.push_back(row[k].y);
    }
    if (!row.empty()) ptr.push_back((int32_t)px.size());
    if (ocol.size() >= (size_t)INT32_MAX || px.size() >= (size_t)INT32_MAX) { *err = "a Galerkin product has 2^31 or more nonzeros or terms (int32 indices)"; return; }
    orowptr[i + 1] = (int32_t)ocol.size();
  }
}

void pair_values(const std::vector<int32_t>& ptr, const std::vector<int32_t>& px, const std::vector<int32_t>& py, const std::vector<double>& X,
                 const std::vector<double>& Y, std::vector<double>& out) {
  out.assign(ptr.size() - 1, 0.0);
  for (size_t q = 0; q + 1 < ptr.size(); ++q) {
    double s = 0.0;
    for (int32_t t = ptr[q]; t < ptr[q + 1]; ++t) s = std::fma(X[px[t]], Y[py[t]], s);
    out[q] = s;
  }
}

// P pattern and values (the device formula), R = P' with its gather map
void interpolation(HostLevel& L, const std::vector<char>& strong, const std::vector<int32_t>& cf) {
  const int32_t n = L.n;
  std::vector<int32_t> cidx(n, -1);
  int32_t nc = 0;
  for (int32_t i = 0; i < n; ++i)
    if (cf[i]) cidx[i] = nc++;
  L.prowptr.assign(n + 1, 0); L.pcol.clear(); L.pmap.clear(); L.pval.clear();
  for (int32_t i = 0; i < n; ++i) {
    if (cf[i]) {
      L.pcol.push_back(cidx[i]); L.pmap.push_back(-1); L.pval.push_back(1.0);
    } else {
      const size_t s0 = L.pcol.size();
      double an = 0.0, ap = 0.0, sn = 0.0, sp = 0.0;
      for (int32_t q = L.rowptr[i]; q < L.rowptr[i + 1]; ++q) {
        if (L.col[q] == i) continue;
        const double v = L.val[q];
        if (v < 0.0) an += v; else if (v > 0.0) ap += v;
        if (strong[q] && cf[L.col[q]]) {
          L.pcol.push_back(cidx[L.col[q]]); L.pmap.push_back(q);
          if (v < 0.0) sn += v; else if (v > 0.0) sp += v;
        }
      }
      double d = L.val[L.diag[i]];
      const double alpha = sn != 0.0 ? an / sn : 0.0;
      double beta = 0.0;
      if (sp == 0.0) d += ap; else beta = ap / sp;
      for (size_t t = s0; t < L.pcol.size(); ++t) {
        const double v = L.val[L.pmap[t]];
        L.pval.push_back(-((v < 0.0 ? alpha : beta) * v) / d);
      }
    }
    L.prowptr[i + 1] = (int32_t)L.pcol.size();
  }
  L.rrowptr.assign(nc + 1, 0);
  for (int32_t t = 0; t < L.prowptr[n]; ++t) L.rrowptr[L.pcol[t] + 1]++;
  for (int32_t c = 0; c < nc; ++c) L.rrowptr[c + 1] += L.rrowptr[c];
  L.rcol.resize(L.prowptr[n]); L.rmap.resize(L.prowptr[n]);
  std::vector<int32_t> fill(L.rrowptr.begin(), L.rrowptr.end() - 1);
  for (int32_t i = 0; i < n; ++i)
    for (int32_t t = L.prowptr[i]; t < L.prowptr[i + 1]; ++t) {
      const int32_t k = fill[L.pcol[t]]++;
      L.rcol[k] = i; L.rmap[k] = t;
    }
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

// the host rebuild: every level's pattern and pair lists, then the upload
int32_t rebuild(b200_amg* amg, const double* nzval) {
  b200_ctx* ctx = amg->ctx;
  const b200_amg_opts& o = amg->o;
  std::vector<double> nz(amg->nnz);
  CUDA_TRY(ctx, cudaMemcpyAsync(nz.data(), nzval, sizeof(double) * amg->nnz, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  std::vector<HostLevel> H(1);
  H[0].n = (int32_t)amg->n;
  H[0].rowptr = amg->rowptr0; H[0].col = amg->col0;
  H[0].val.resize(amg->nnz);
  for (int64_t q = 0; q < amg->nnz; ++q) H[0].val[q] = nz[amg->map0[q]];
  for (;;) {
    HostLevel& L = H.back();
    L.diag.assign(L.n, -1);
    for (int32_t i = 0; i < L.n; ++i)
      for (int32_t q = L.rowptr[i]; q < L.rowptr[i + 1]; ++q)
        if (L.col[q] == i) L.diag[i] = q;
    if (L.n <= o.max_coarse || (int32_t)H.size() >= o.max_levels) break;
    std::vector<char> strong;
    std::vector<int32_t> cf;
    strength(L.n, L.rowptr, L.col, L.val.data(), o.theta, strong);
    const int64_t nc = rs_split(L.n, L.rowptr, L.col, strong, cf);
    if (nc == 0 || nc == L.n) break;
    interpolation(L, strong, cf);
    const char* err = nullptr;
    std::vector<double> apval, rval(L.rcol.size()), acval;
    for (size_t k = 0; k < L.rcol.size(); ++k) rval[k] = L.pval[L.rmap[k]];
    pair_product(L.n, L.rowptr, L.col, L.prowptr, L.pcol, L.ap_rowptr, L.ap_col, L.ap_ptr, L.ap_x, L.ap_y, &err);
    if (err) return ctx->fail(B200_ERR_UNSUPPORTED, err, __FILE__, __LINE__);
    pair_values(L.ap_ptr, L.ap_x, L.ap_y, L.val, L.pval, apval);
    HostLevel Cl;
    Cl.n = (int32_t)nc;
    pair_product(Cl.n, L.rrowptr, L.rcol, L.ap_rowptr, L.ap_col, Cl.rowptr, Cl.col, L.ac_ptr, L.ac_x, L.ac_y, &err);
    if (err) return ctx->fail(B200_ERR_UNSUPPORTED, err, __FILE__, __LINE__);
    pair_values(L.ac_ptr, L.ac_x, L.ac_y, rval, apval, Cl.val);
    H.push_back(std::move(Cl));
  }
  const int64_t nco = H.back().n;
  if (nco > AMG_DENSE_CAP) {
    char msg[256];
    snprintf(msg, sizeof(msg), "amg_setup: the hierarchy ends at %lld unknowns (%zu levels), above the %lld of the coarsest level's dense inverse: raise max_levels",
             (long long)nco, H.size(), (long long)AMG_DENSE_CAP);
    return ctx->fail(B200_ERR_UNSUPPORTED, msg, __FILE__, __LINE__);
  }
  free_hierarchy(amg);
  bool ok = true;
  auto up = [&](int32_t** d, const std::vector<int32_t>& h) {
    if (!ok) return;
    ok = cudaMalloc(d, sizeof(int32_t) * std::max<size_t>(h.size(), 1)) == cudaSuccess;
    if (ok) amg->owned.push_back(*d);
    if (ok && !h.empty()) ok = cudaMemcpyAsync(*d, h.data(), sizeof(int32_t) * h.size(), cudaMemcpyHostToDevice, ctx->stream) == cudaSuccess;
  };
  auto alloc = [&](double** d, size_t count) {
    if (!ok) return;
    ok = cudaMalloc(d, sizeof(double) * std::max<size_t>(count, 1)) == cudaSuccess;
    if (ok) amg->owned.push_back(*d);
  };
  amg->lev.resize(H.size());
  for (size_t l = 0; l < H.size(); ++l) {
    HostLevel& h = H[l];
    AmgLevel& L = amg->lev[l];
    L.n = h.n; L.nnz = h.rowptr[h.n];
    up(&L.rowptr, h.rowptr); up(&L.col, h.col); up(&L.diag, h.diag);
    alloc(&L.val, L.nnz); alloc(&L.dinv, L.n);
    alloc(&L.x, L.n); alloc(&L.x2, L.n); alloc(&L.b, L.n); alloc(&L.r, L.n);
    if (l + 1 < H.size()) {
      L.pnnz = h.prowptr[h.n]; L.apnnz = (int32_t)h.ap_col.size();
      up(&L.prowptr, h.prowptr); up(&L.pcol, h.pcol); up(&L.pmap, h.pmap); alloc(&L.pval, L.pnnz);
      up(&L.rrowptr, h.rrowptr); up(&L.rcol, h.rcol); up(&L.rmap, h.rmap); alloc(&L.rval, L.pnnz);
      alloc(&L.apval, L.apnnz);
      up(&L.ap_ptr, h.ap_ptr); up(&L.ap_x, h.ap_x); up(&L.ap_y, h.ap_y);
      up(&L.ac_ptr, h.ac_ptr); up(&L.ac_x, h.ac_x); up(&L.ac_y, h.ac_y);
    }
  }
  alloc(&amg->d_dense, (size_t)nco * nco);
  alloc(&amg->d_ainv, (size_t)nco * nco);
  if (ok) {
    ok = cudaMalloc(&amg->d_ipiv, sizeof(int64_t) * nco) == cudaSuccess;
    if (ok) amg->owned.push_back(amg->d_ipiv);
  }
  ok = ok && cudaStreamSynchronize(ctx->stream) == cudaSuccess;  // the host vectors die at scope exit
  if (!ok) {
    cudaGetLastError();
    free_hierarchy(amg);
    return ctx->fail(B200_ERR_NOMEM, "AMG: the hierarchy does not fit in device memory", __FILE__, __LINE__);
  }
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
  for (int32_t l = 0; l + 1 < nlev; ++l) {
    AmgLevel &L = amg->lev[l], &Cl = amg->lev[l + 1];
    LAUNCH(ctx, amg_interp_kernel, blocks(L.n), AT, 0, L.n, (const int32_t*)L.rowptr, (const int32_t*)L.col, (const int32_t*)L.diag, (const double*)L.val,
           (const int32_t*)L.prowptr, (const int32_t*)L.pmap, L.pval, l, amg->d_info);
    LAUNCH(ctx, amg_gather_kernel, blocks(L.pnnz), AT, 0, L.pnnz, (const int32_t*)L.rmap, (const double*)L.pval, L.rval);
    LAUNCH(ctx, amg_pair_product_kernel, blocks(L.apnnz), AT, 0, L.apnnz, (const int32_t*)L.ap_ptr, (const int32_t*)L.ap_x, (const int32_t*)L.ap_y,
           (const double*)L.val, (const double*)L.pval, L.apval);
    LAUNCH(ctx, amg_pair_product_kernel, blocks(Cl.nnz), AT, 0, Cl.nnz, (const int32_t*)L.ac_ptr, (const int32_t*)L.ac_x, (const int32_t*)L.ac_y,
           (const double*)L.rval, (const double*)L.apval, Cl.val);
    LAUNCH(ctx, amg_dinv_kernel, blocks(L.n), AT, 0, L.n, (const int32_t*)L.diag, (const double*)L.val, L.dinv, l, amg->d_info);
  }
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
  B200_REQUIRE(ctx, n > 0 && colptr && rowval && out && (base == 0 || base == 1), "amg_create: bad arguments");
  const int64_t nnz = colptr[n] - colptr[0];
  B200_REQUIRE(ctx, colptr[0] == base && nnz >= 0, "amg_create: colptr must start at the index base");
  B200_REQUIRE(ctx, n < INT32_MAX && nnz < INT32_MAX, "amg_create: n and nnz must be below 2^31 (int32 CSR indices)");
  b200_amg_opts o;
  b200_amg_opts_default(&o);
  if (opts) o = *opts;
  B200_REQUIRE(ctx, o.theta >= 0.0 && o.theta <= 1.0 && o.omega > 0.0 && o.presweeps >= 0 && o.postsweeps >= 0 && o.max_levels >= 1 && o.max_coarse >= 1,
               "amg_create: options out of range (0 <= theta <= 1, omega > 0, sweeps >= 0, max_levels >= 1, max_coarse >= 1)");
  std::vector<int32_t> rowptr, col, map, diag;
  const std::string err = b200i_csr_of_csc("amg_create", n, colptr, rowval, base, true, rowptr, col, map, diag);
  if (!err.empty()) return ctx->fail(B200_ERR_INVALID, err.c_str(), __FILE__, __LINE__);
  b200_amg* amg = new b200_amg();
  amg->ctx = ctx; amg->n = n; amg->nnz = nnz; amg->o = o;
  amg->rowptr0 = std::move(rowptr); amg->col0 = std::move(col); amg->map0 = std::move(map);
  bool ok = cudaMalloc(&amg->d_map0, sizeof(int32_t) * std::max<int64_t>(nnz, 1)) == cudaSuccess && cudaMalloc(&amg->d_info, sizeof(int32_t)) == cudaSuccess &&
            (nnz == 0 || cudaMemcpyAsync(amg->d_map0, amg->map0.data(), sizeof(int32_t) * nnz, cudaMemcpyHostToDevice, ctx->stream) == cudaSuccess) &&
            cudaStreamSynchronize(ctx->stream) == cudaSuccess;
  if (!ok) { cudaGetLastError(); b200_amg_destroy(amg); return ctx->fail(B200_ERR_NOMEM, "AMG: out of device memory", __FILE__, __LINE__); }
  *out = amg;
  return B200_OK;
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
  B200_REQUIRE(ctx, amg->refreshed && rowptr && level >= 0 && level < nlev && (what == B200_AMG_EXPORT_A || (what == B200_AMG_EXPORT_P && level + 1 < nlev)),
               "amg_export: bad arguments (P exists on every level but the coarsest), or no setup yet");
  const AmgLevel& L = amg->lev[level];
  const bool a = what == B200_AMG_EXPORT_A;
  const int32_t nz = a ? L.nnz : L.pnnz;
  CUDA_TRY(ctx, cudaMemcpyAsync(rowptr, a ? L.rowptr : L.prowptr, sizeof(int32_t) * (L.n + 1), cudaMemcpyDeviceToHost, ctx->stream));
  if (col) CUDA_TRY(ctx, cudaMemcpyAsync(col, a ? L.col : L.pcol, sizeof(int32_t) * nz, cudaMemcpyDeviceToHost, ctx->stream));
  if (val) CUDA_TRY(ctx, cudaMemcpyAsync(val, a ? L.val : L.pval, sizeof(double) * nz, cudaMemcpyDeviceToHost, ctx->stream));
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
