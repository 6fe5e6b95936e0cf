// ilu0.cu — ILU(0) of an assembled sparse matrix and its triangular solve, the algebraic preconditioner of GMRES on the
// sparse route (`KrylovJL_GMRES(precs = ...)` with an incomplete LU of W, docs/src/tutorials/large_systems.md:244-316).
//
//   * symbolic phase (host, once per pattern): the CSR view of the CSC pattern (int32 indices), the diagonal position of
//     every row, and the level sets of the strictly lower pattern (forward sweep, also the factorisation order) and of the
//     strictly upper pattern (backward sweep).  Row i of a level depends only on rows of earlier levels;
//   * numeric factorisation (device, every fresh Jacobian): gather the CSC values into CSR order, then row-wise IKJ ILU(0)
//     — for each lower k of row i in ascending order: a_ik /= u_kk, a_ij -= a_ik u_kj for every j > k in row i's pattern —
//     one warp per row, all levels in ONE cooperative launch with a grid barrier between levels.  u_kj is found by a binary
//     search of row k's sorted upper part by the lane that owns a_ij (no position map: it would cost nnz x row-length int32
//     entries, ~128 MB at 3D N = 100, and the rows here are short);
//   * apply: x = U^-1 L^-1 b (L unit lower), forward then backward level sweeps, one warp per row, one cooperative launch.
// Every row's operations run in a fixed order (lane-strided partial sums, a fixed butterfly), so factors and solves are
// bit-reproducible.  Values written inside a launch are read back with ordinary (coherent) loads after the grid barrier.
#include "common.cuh"
#include <cooperative_groups.h>
#include <algorithm>
#include <climits>
#include <vector>

namespace cg = cooperative_groups;

struct b200_ilu0 {
  b200_ctx* ctx;
  int64_t n, nnz;
  int32_t nlev_lower, nlev_upper;
  int32_t *d_rowptr, *d_col, *d_map, *d_diag;  // CSR view; map: CSR position -> caller's CSC position
  int32_t *d_lrows, *d_lptr, *d_urows, *d_uptr; // rows ordered by level, level pointers
  double* d_lu;                                 // packed factors in CSR order
  int32_t* d_info;
  int grid;                                     // CTAs of the cooperative launches
  int factored;
};

namespace {
constexpr int IL_THREADS = 256;
constexpr int IL_WARPS = IL_THREADS / 32;

struct IluParams {
  int64_t n;
  const int32_t *rowptr, *col, *diag;
  const int32_t *lrows, *lptr, *urows, *uptr;
  int32_t nlev_lower, nlev_upper;
};

__global__ void ilu_gather_kernel(int64_t nnz, const int32_t* __restrict__ map, const double* __restrict__ nzval, double* __restrict__ lu) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q < nnz) lu[q] = nzval[map[q]];
}
__global__ void ilu_scatter_kernel(int64_t nnz, const int32_t* __restrict__ map, const double* __restrict__ lu, double* __restrict__ out) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q < nnz) out[map[q]] = lu[q];
}

// position of column j in the sorted range col[lo, hi), or -1
__device__ __forceinline__ int32_t find_col(const int32_t* col, int32_t lo, int32_t hi, int32_t j) {
  while (lo < hi) {
    const int32_t mid = (lo + hi) >> 1;
    const int32_t c = col[mid];
    if (c == j) return mid;
    if (c < j) lo = mid + 1; else hi = mid;
  }
  return -1;
}

// a / b, correctly rounded whenever the quotient, b and 1/b are normal numbers (Markstein: a correctly rounded reciprocal and one
// fma correction of a faithful quotient).  The division operator would call its slow-path subroutine, whose register saves are
// spills in this kernel.
__device__ __forceinline__ double quot(double a, double b) {
  const double r = __drcp_rn(b);
  const double q = a * r;
  return fma(r, fma(-b, q, a), q);
}

// IKJ ILU(0) of all rows, level by level; *info = smallest 1-based row whose pivot u_ii is zero or not finite (0: none)
__global__ void __launch_bounds__(IL_THREADS) ilu0_factor_kernel(IluParams P, double* lu, int32_t* info) {
  cg::grid_group grid = cg::this_grid();
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int32_t l = 0; l < P.nlev_lower; ++l) {
    for (int64_t t = P.lptr[l] + warp; t < P.lptr[l + 1]; t += nwarps) {
      const int32_t i = P.lrows[t];
      const int32_t beg = P.rowptr[i], end = P.rowptr[i + 1], di = P.diag[i];
      for (int32_t pk = beg; pk < di; ++pk) {
        const int32_t k = P.col[pk];
        const double lik = quot(lu[pk], lu[P.diag[k]]);
        const int32_t ku0 = P.diag[k] + 1, ku1 = P.rowptr[k + 1];
        for (int32_t q = pk + 1 + lane; q < end; q += 32) {
          const int32_t pos = find_col(P.col, ku0, ku1, P.col[q]);
          if (pos >= 0) lu[q] = fma(-lik, lu[pos], lu[q]);
        }
        __syncwarp();
        if (lane == 0) lu[pk] = lik;
        __syncwarp();
      }
      if (lane == 0) {
        const double d = lu[di];
        if (d == 0.0 || !isfinite(d)) atomicMin(info, i + 1);
      }
    }
    grid.sync();
  }
}

// x = U^-1 L^-1 b; x may alias b (row i reads b_i before it writes x_i, and no other row reads b_i)
__global__ void __launch_bounds__(IL_THREADS) ilu0_solve_kernel(IluParams P, const double* lu, const double* b, double* x) {
  cg::grid_group grid = cg::this_grid();
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int32_t l = 0; l < P.nlev_lower; ++l) {  // forward: y_i = b_i - sum_{j < i} l_ij y_j
    for (int64_t t = P.lptr[l] + warp; t < P.lptr[l + 1]; t += nwarps) {
      const int32_t i = P.lrows[t];
      const int32_t beg = P.rowptr[i], di = P.diag[i];
      double s = 0.0;
      for (int32_t q = beg + lane; q < di; q += 32) s = fma(lu[q], x[P.col[q]], s);
      s = warp_sum(s);
      if (lane == 0) x[i] = b[i] - s;
    }
    grid.sync();
  }
  for (int32_t l = 0; l < P.nlev_upper; ++l) {  // backward: x_i = (y_i - sum_{j > i} u_ij x_j) / u_ii
    for (int64_t t = P.uptr[l] + warp; t < P.uptr[l + 1]; t += nwarps) {
      const int32_t i = P.urows[t];
      const int32_t di = P.diag[i], end = P.rowptr[i + 1];
      double s = 0.0;
      for (int32_t q = di + 1 + lane; q < end; q += 32) s = fma(lu[q], x[P.col[q]], s);
      s = warp_sum(s);
      if (lane == 0) x[i] = (x[i] - s) / lu[di];
    }
    if (l + 1 < P.nlev_upper) grid.sync();
  }
}

// level of every row from its dependencies (lower: j < i, rows ascending; upper: j > i, rows descending), then the rows
// grouped by level (ascending row index inside a level) with level pointers
void level_sets(int64_t n, const std::vector<int32_t>& rowptr, const std::vector<int32_t>& col, const std::vector<int32_t>& diag, bool lower,
                std::vector<int32_t>& rows, std::vector<int32_t>& ptr) {
  std::vector<int32_t> lev(n, 0);
  int32_t nlev = 0;
  for (int64_t s = 0; s < n; ++s) {
    const int64_t i = lower ? s : n - 1 - s;
    int32_t L = 0;
    const int32_t q0 = lower ? rowptr[i] : diag[i] + 1, q1 = lower ? diag[i] : rowptr[i + 1];
    for (int32_t q = q0; q < q1; ++q) L = std::max(L, lev[col[q]] + 1);
    lev[i] = L;
    nlev = std::max(nlev, L + 1);
  }
  ptr.assign(nlev + 1, 0);
  for (int64_t i = 0; i < n; ++i) ptr[lev[i] + 1]++;
  for (int32_t l = 0; l < nlev; ++l) ptr[l + 1] += ptr[l];
  rows.resize(n);
  std::vector<int32_t> fill(ptr.begin(), ptr.end() - 1);
  for (int64_t i = 0; i < n; ++i) rows[fill[lev[i]]++] = (int32_t)i;
}

IluParams params(const b200_ilu0* ilu) {
  IluParams P;
  P.n = ilu->n; P.rowptr = ilu->d_rowptr; P.col = ilu->d_col; P.diag = ilu->d_diag;
  P.lrows = ilu->d_lrows; P.lptr = ilu->d_lptr; P.urows = ilu->d_urows; P.uptr = ilu->d_uptr;
  P.nlev_lower = ilu->nlev_lower; P.nlev_upper = ilu->nlev_upper;
  return P;
}
}  // namespace

std::string b200i_csr_of_csc(const char* who, int64_t n, const int64_t* colptr, const int64_t* rowval, int32_t base, bool require_diag,
                             std::vector<int32_t>& rowptr, std::vector<int32_t>& col, std::vector<int32_t>& map, std::vector<int32_t>& diag) {
  const int64_t nnz = colptr[n] - colptr[0];
  char msg[200];
  // CSR view: walking the columns in order leaves every row's column indices ascending
  rowptr.assign(n + 1, 0); col.assign(nnz, 0); map.assign(nnz, 0); diag.assign(n, -1);
  for (int64_t c = 0; c < n; ++c) {
    if (colptr[c + 1] < colptr[c]) { snprintf(msg, sizeof(msg), "%s: colptr must be non-decreasing", who); return msg; }
    for (int64_t p = colptr[c] - base; p < colptr[c + 1] - base; ++p) {
      const int64_t r = rowval[p] - base;
      if (r < 0 || r >= n) { snprintf(msg, sizeof(msg), "%s: row index out of range", who); return msg; }
      rowptr[r + 1]++;
    }
  }
  for (int64_t r = 0; r < n; ++r) rowptr[r + 1] += rowptr[r];
  {
    std::vector<int32_t> fill(rowptr.begin(), rowptr.end() - 1);
    for (int64_t c = 0; c < n; ++c)
      for (int64_t p = colptr[c] - base; p < colptr[c + 1] - base; ++p) {
        const int32_t q = fill[rowval[p] - base]++;
        col[q] = (int32_t)c; map[q] = (int32_t)p;
      }
  }
  for (int64_t r = 0; r < n; ++r) {
    for (int32_t q = rowptr[r]; q < rowptr[r + 1]; ++q) {
      if (q > rowptr[r] && col[q] == col[q - 1]) {
        snprintf(msg, sizeof(msg), "%s: duplicate entry (%lld, %lld) in the pattern", who, (long long)(r + base), (long long)(col[q] + base));
        return msg;
      }
      if (col[q] == r) diag[r] = q;
    }
    if (require_diag && diag[r] < 0) {
      snprintf(msg, sizeof(msg), "%s: row %lld (index base %d) has no structural diagonal entry", who, (long long)(r + base), (int)base);
      return msg;
    }
  }
  return std::string();
}

extern "C" {
int32_t b200_ilu0_destroy(b200_ilu0* ilu) {
  if (!ilu) return B200_OK;
  B200_DEVICE_GUARD(ilu->ctx);
  cudaStreamSynchronize(ilu->ctx->stream);
  cudaFree(ilu->d_rowptr); cudaFree(ilu->d_col); cudaFree(ilu->d_map); cudaFree(ilu->d_diag);
  cudaFree(ilu->d_lrows); cudaFree(ilu->d_lptr); cudaFree(ilu->d_urows); cudaFree(ilu->d_uptr);
  cudaFree(ilu->d_lu); cudaFree(ilu->d_info);
  delete ilu;
  return B200_OK;
}

int32_t b200_ilu0_create(b200_ctx* ctx, int64_t n, const int64_t* colptr, const int64_t* rowval, int32_t base, b200_ilu0** out) {
  B200_DEVICE_GUARD(ctx);
  B200_REQUIRE(ctx, n > 0 && colptr && rowval && out && (base == 0 || base == 1), "ilu0_create: bad arguments");
  const int64_t nnz = colptr[n] - colptr[0];
  B200_REQUIRE(ctx, colptr[0] == base && nnz >= 0, "ilu0_create: colptr must start at the index base");
  B200_REQUIRE(ctx, n < INT32_MAX && nnz < INT32_MAX, "ilu0_create: n and nnz must be below 2^31 (int32 CSR indices)");
  std::vector<int32_t> rowptr, col, map, diag;
  const std::string err = b200i_csr_of_csc("ilu0_create", n, colptr, rowval, base, true, rowptr, col, map, diag);
  if (!err.empty()) return ctx->fail(B200_ERR_INVALID, err.c_str(), __FILE__, __LINE__);
  std::vector<int32_t> lrows, lptr, urows, uptr;
  level_sets(n, rowptr, col, diag, true, lrows, lptr);
  level_sets(n, rowptr, col, diag, false, urows, uptr);
  int32_t width = 1;
  for (size_t l = 0; l + 1 < lptr.size(); ++l) width = std::max(width, lptr[l + 1] - lptr[l]);
  for (size_t l = 0; l + 1 < uptr.size(); ++l) width = std::max(width, uptr[l + 1] - uptr[l]);
  // cooperative grid: no more CTAs than co-reside, nor than the widest level has rows for (one warp per row)
  int per_sm_f = 0, per_sm_s = 0;
  CUDA_TRY(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_f, ilu0_factor_kernel, IL_THREADS, 0));
  CUDA_TRY(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_s, ilu0_solve_kernel, IL_THREADS, 0));
  const int per_sm = std::min(per_sm_f, per_sm_s);
  B200_REQUIRE(ctx, per_sm > 0, "ilu0_create: the level kernels cannot be resident");
  b200_ilu0* ilu = new b200_ilu0();
  memset(ilu, 0, sizeof(*ilu));
  ilu->ctx = ctx; ilu->n = n; ilu->nnz = nnz;
  ilu->nlev_lower = (int32_t)lptr.size() - 1; ilu->nlev_upper = (int32_t)uptr.size() - 1;
  ilu->grid = (int)std::min<int64_t>((int64_t)per_sm * ctx->sm_count, (width + IL_WARPS - 1) / IL_WARPS);
  auto up = [&](int32_t** d, const std::vector<int32_t>& h) -> bool {
    if (cudaMalloc(d, sizeof(int32_t) * std::max<size_t>(h.size(), 1)) != cudaSuccess) return false;
    return h.empty() || cudaMemcpyAsync(*d, h.data(), sizeof(int32_t) * h.size(), cudaMemcpyHostToDevice, ctx->stream) == cudaSuccess;
  };
  bool ok = up(&ilu->d_rowptr, rowptr) && up(&ilu->d_col, col) && up(&ilu->d_map, map) && up(&ilu->d_diag, diag) &&
            up(&ilu->d_lrows, lrows) && up(&ilu->d_lptr, lptr) && up(&ilu->d_urows, urows) && up(&ilu->d_uptr, uptr) &&
            cudaMalloc(&ilu->d_lu, sizeof(double) * std::max<int64_t>(nnz, 1)) == cudaSuccess && cudaMalloc(&ilu->d_info, sizeof(int32_t)) == cudaSuccess &&
            cudaStreamSynchronize(ctx->stream) == cudaSuccess;  // the host vectors die at scope exit
  if (!ok) { cudaGetLastError(); b200_ilu0_destroy(ilu); return ctx->fail(B200_ERR_NOMEM, "ILU(0): out of device memory", __FILE__, __LINE__); }
  *out = ilu;
  return B200_OK;
}

int32_t b200_ilu0_levels(b200_ilu0* ilu, int32_t* lower, int32_t* upper) {
  if (lower) *lower = ilu->nlev_lower;
  if (upper) *upper = ilu->nlev_upper;
  return B200_OK;
}

int32_t b200_ilu0_factor(b200_ilu0* ilu, const double* nzval, int32_t* info_host) {
  B200_DEVICE_GUARD(ilu ? ilu->ctx : nullptr);
  b200_ctx* ctx = ilu->ctx;
  B200_REQUIRE(ctx, nzval, "ilu0_factor: bad arguments");
  const int32_t none = INT_MAX;
  CUDA_TRY(ctx, cudaMemcpyAsync(ilu->d_info, &none, sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
  LAUNCH(ctx, ilu_gather_kernel, (int)((ilu->nnz + 255) / 256), 256, 0, ilu->nnz, (const int32_t*)ilu->d_map, nzval, ilu->d_lu);
  B200_TRY(coop_launch(ctx, B200_KID_SPARSE, 0.0, ilu0_factor_kernel, ilu->grid, IL_THREADS, 0, params(ilu), ilu->d_lu, ilu->d_info));
  int32_t h = 0;
  CUDA_TRY(ctx, cudaMemcpyAsync(&h, ilu->d_info, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  ilu->factored = 1;
  if (info_host) *info_host = h == INT_MAX ? 0 : h;
  return B200_OK;
}

int32_t b200_ilu0_solve(b200_ilu0* ilu, const double* b, double* x) {
  B200_DEVICE_GUARD(ilu ? ilu->ctx : nullptr);
  b200_ctx* ctx = ilu->ctx;
  B200_REQUIRE(ctx, ilu->factored, "ilu0_solve before ilu0_factor");
  return coop_launch(ctx, B200_KID_SPARSE, 12.0 * (double)ilu->nnz + 3.0 * 8.0 * (double)ilu->n, ilu0_solve_kernel, ilu->grid, IL_THREADS, 0, params(ilu),
                     ilu->d_lu, b, x);
}

int32_t b200_ilu0_export(b200_ilu0* ilu, double* nzval_out) {
  B200_DEVICE_GUARD(ilu ? ilu->ctx : nullptr);
  b200_ctx* ctx = ilu->ctx;
  B200_REQUIRE(ctx, ilu->factored && nzval_out, "ilu0_export: bad arguments or not factored");
  LAUNCH(ctx, ilu_scatter_kernel, (int)((ilu->nnz + 255) / 256), 256, 0, ilu->nnz, (const int32_t*)ilu->d_map, (const double*)ilu->d_lu, nzval_out);
  CHECK_LAUNCH(ctx);
  return B200_OK;
}

int32_t b200_ilu0_linop(b200_ilu0* ilu, b200_linop** out) {
  B200_DEVICE_GUARD(ilu ? ilu->ctx : nullptr);
  B200_REQUIRE(ilu->ctx, out, "ilu0_linop: bad arguments");
  b200_linop* op = new b200_linop();
  memset(op, 0, sizeof(*op));
  op->ctx = ilu->ctx; op->kind = LINOP_ILU0; op->n = ilu->n; op->ilu = ilu;
  *out = op;
  return B200_OK;
}
}  // extern "C"
