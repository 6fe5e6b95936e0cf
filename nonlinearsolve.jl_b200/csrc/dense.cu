// dense.cu — dense Jacobian fallback (SURVEY.md §8a row a5; kernels K7, K8): analytic fill of the column-major n x n
// Jacobian and a two-level blocked right-looking LU with partial pivoting (LAPACK getrf/getrs semantics).
//
// Reference path replaced: JacobianCache call lib/NonlinearSolveBase/src/jacobian.jl:237-258 (DI.jacobian! with dense
// AutoForwardDiff: exact derivatives) and the LinearSolve LU reached through linear_solve.jl:100-117 /
// NonlinearSolveBaseLinearSolveExt.jl:16-32, 102-111 (copyto!(A, J); lu!; ldiv!).
//
// getrf structure (outer block NBO = 256 / 512, inner block NBI = 32):
//   inner panel (32 columns): ONE cooperative kernel (`panel_coop_kernel`): every CTA keeps its rows of the panel in shared
//       memory for all 32 columns; per column only the arg-max partials and two 32-double rows cross CTAs
//   after an inner panel: TRSM (`u12_fused_kernel`) + GEMM (K = 32) on the remaining columns of the outer panel
//   after the outer panel: row interchanges applied to the columns left/right of it, TRSM for U12 (`u12_fused_kernel`), and
//       the trailing update  A22 -= L21 U12  with K = NBO — the GEMM-shaped 2/3 n^3 flops — on the FP64 tensor cores
//       (`gemm_sub_w8_kernel`: mma.sync.m8n8k4.f64 = DMMA.8x8x4 in SASS, the native FP64 MMA shape of sm_90a — m16n8k16
//       compiles to eight of them; wgmma has no FP64 kind).  Look-ahead: the next panel's columns are updated first and
//       the panel is factored on a second, HIGHEST-PRIORITY stream underneath the rest of the update.
// Pivot rule is LAPACK's (largest magnitude, first index wins ties).  tests/test_gpu_dense_lu.py checks the factorisation in
// every blocking regime up to n = 32768: LAPACK's pivots up to its first ambiguous column and on exactly constructed ties,
// |L| <= 1, Higham's componentwise error bounds for getrf and getrs, info on exactly zero columns, and bit-identical repeats.
#include "common.cuh"
#include <math.h>
#include <algorithm>

namespace {
constexpr int NBO_DEFAULT = 256;  // outer block (GEMM K)
constexpr int NBI = 32;   // inner panel width
constexpr int DT = 256;
constexpr int PS_MAX = 160;  // max CTAs of the panel grids

// ------------------------------------------------------------------ Jacobian fill
__global__ void __launch_bounds__(DT) bruss_dense_fill_kernel(int dim, int N, double a, double A, const double* __restrict__ u,
                                                               double* __restrict__ J, int64_t ld) {
  const int64_t N2 = (int64_t)N * N, NC = (dim == 2) ? N2 : N2 * N, n = 2 * NC;
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;  // column
  if (c >= n) return;
  const int s = (int)(c / NC);
  const int64_t cell = c - (int64_t)s * NC;
  const int i = (int)(cell % N), j = (int)((cell / N) % N), k = (dim == 3) ? (int)(cell / N2) : 0;
  const int ip = (i + 1 == N) ? 0 : i + 1, im = (i == 0) ? N - 1 : i - 1;
  const int jp = (j + 1 == N) ? 0 : j + 1, jm = (j == 0) ? N - 1 : j - 1;
  const int kp = (k + 1 == N) ? 0 : k + 1, km = (k == 0) ? N - 1 : k - 1;
  const double uc = u[cell], vc = u[cell + NC];
  const double diag_lap = (dim == 2) ? -4.0 * a : -6.0 * a;
  double dself, dcross;
  if (s == 0) { dself = 2.0 * uc * vc - (A + 1.0); dcross = A - 2.0 * uc * vc; }
  else { dself = -(uc * uc); dcross = uc * uc; }
  double* col = J + c * ld;
  const int64_t off = (int64_t)s * NC, offx = (int64_t)(1 - s) * NC;
  // neighbours first (+=, they may coincide for tiny N), column was zeroed by the caller
  col[im + (int64_t)N * j + N2 * k + off] += a;
  col[ip + (int64_t)N * j + N2 * k + off] += a;
  col[i + (int64_t)N * jm + N2 * k + off] += a;
  col[i + (int64_t)N * jp + N2 * k + off] += a;
  if (dim == 3) {
    col[i + (int64_t)N * j + N2 * km + off] += a;
    col[i + (int64_t)N * j + N2 * kp + off] += a;
  }
  col[cell + off] += diag_lap + dself;
  col[cell + offx] += dcross;
}
__global__ void __launch_bounds__(DT) small_dense_fill_kernel(int kind, int64_t n, const double* __restrict__ u, double* __restrict__ J, int64_t ld) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n) return;
  double* col = J + c * ld;
  if (kind == 0) {
    col[c] = 2.0 * u[c];
  } else {  // F_i = u_i + 0.1 u_i (2 u_i - u_{i-1} - u_{i+1}) - p_i
    double t = 2.0 * u[c];
    if (c > 0) t -= u[c - 1];
    if (c + 1 < n) t -= u[c + 1];
    col[c] = 1.0 + 0.1 * (t + 2.0 * u[c]);
    if (c > 0) col[c - 1] = -0.1 * u[c - 1];
    if (c + 1 < n) col[c + 1] = -0.1 * u[c + 1];
  }
}
__global__ void __launch_bounds__(DT) unit_vector_kernel(int64_t n, int64_t j, double* __restrict__ e) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) e[i] = (i == j) ? 1.0 : 0.0;
}

// ------------------------------------------------------------------ panel factorisation (multi-CTA, column by column)
__device__ __forceinline__ void argmax_combine(double& best, int64_t& bidx, double ob, int64_t oi) {
  // LAPACK idamax: largest |value|, first index wins ties; a NaN encountered first stays
  if (ob > best || (ob == best && oi < bidx)) { best = ob; bidx = oi; }
}
__device__ __forceinline__ void block_argmax(double& best, int64_t& bidx, double* smax, int64_t* sidx) {
  for (int o = 16; o > 0; o >>= 1) {
    const double ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int64_t oi = __shfl_xor_sync(0xffffffffu, bidx, o);
    argmax_combine(best, bidx, ob, oi);
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
  if (lane == 0) { smax[wid] = best; sidx[wid] = bidx; }
  __syncthreads();
  if (wid == 0) {
    best = (lane < nw) ? smax[lane] : -2.0;
    bidx = (lane < nw) ? sidx[lane] : INT64_MAX;
    for (int o = 16; o > 0; o >>= 1) {
      const double ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int64_t oi = __shfl_xor_sync(0xffffffffu, bidx, o);
      argmax_combine(best, bidx, ob, oi);
    }
  }
}

// ---- cooperative inner panel: the kbi (<= 32) columns [c0, c0+kbi), rows [c0, n), factored by ONE kernel.  Every CTA keeps
// its contiguous chunk of panel rows in shared memory (column-major, so a thread-per-row sweep is conflict free) for the
// whole panel.  Per column ONE exchange crosses CTAs, and it carries its own synchronisation (the flag-in-word publication of
// common.cuh, ll_store / ll_load / ll_wait): each CTA publishes {its arg-max, the panel row that holds it} — and CTA 0, which always owns row `col`, that
// row too — then polls the P headers, picks the pivot (LAPACK idamax rule) and reads the winner's row.  This replaces
// two cooperative-groups grid barriers per column (the panel sits on the critical path of the last third of the
// factorisation).  Launched cooperatively for the co-residency guarantee only.
constexpr int PX_HREPL = 16, PX_RREPL = 4;   // replicas of the headers / rows (pollers of CTA b read replica b mod R: spreads the hot lines)
constexpr size_t PX_HDR_WORDS = (size_t)2 * PX_HREPL * PS_MAX * 4;
constexpr size_t PX_ROW_WORDS = (size_t)2 * PX_RREPL * PS_MAX * 2 * NBI * 2;
constexpr size_t PX_WORDS = PX_HDR_WORDS + PX_ROW_WORDS;
__device__ __forceinline__ unsigned long long px_load(const unsigned long long* src, unsigned epoch, int* fault) {
  ulonglong2 p = ll_load(src);
  ll_wait(src, p, epoch, 1u << 24, fault);
  return ll_value(p);
}
__device__ __forceinline__ size_t px_hdr_at(int buf, int rep, int cta) { return (((size_t)buf * PX_HREPL + rep) * PS_MAX + cta) * 4; }
__device__ __forceinline__ size_t px_row_at(int buf, int rep, int cta, int kind, int c) {
  return PX_HDR_WORDS + (((((size_t)buf * PX_RREPL + rep) * PS_MAX + cta) * 2 + kind) * NBI + c) * 2;
}

__global__ void __launch_bounds__(DT) panel_coop_kernel(int64_t n, double* __restrict__ A, int64_t ld, int64_t c0, int kbi, int rpc,
                                                         int64_t* __restrict__ ipiv, int* __restrict__ info, unsigned long long* __restrict__ xw) {
  extern __shared__ double pa[];  // [kbi][rpc_pad]
  __shared__ double urow[NBI];
  __shared__ double smax[32];
  __shared__ int64_t sidx[32];
  __shared__ int64_t piv_s;
  __shared__ int fault_s;
  const int rp = rpc | 1;
  const int b = blockIdx.x, P = gridDim.x, tid = threadIdx.x;
  const int64_t row0 = c0 + (int64_t)b * rpc;          // first global row of this CTA
  const int nrows = (int)max((int64_t)0, min((int64_t)rpc, n - row0));
  if (tid == 0) fault_s = 0;
  for (int c = 0; c < kbi; ++c)
    for (int r = tid; r < nrows; r += DT) pa[c * rp + r] = A[(c0 + c) * ld + row0 + r];
  __syncthreads();
  for (int jj = 0; jj < kbi; ++jj) {
    const int64_t col = c0 + jj;
    const unsigned epoch = (unsigned)(col + 1);
    const int buf = (int)(col & 1);
    // (a) local arg-max of |a[., jj]| over rows >= col
    double best = -1.0;
    int64_t bidx = INT64_MAX;
    for (int r = tid; r < nrows; r += DT) {
      const int64_t gr = row0 + r;
      if (gr >= col) {
        const double v = fabs(pa[jj * rp + r]);
        if (v > best) { best = v; bidx = gr; }
      }
    }
    block_argmax(best, bidx, smax, sidx);  // result in every lane of warp 0
    // (b) publish: the candidate row (and row `col` from its owner, CTA 0), then the header
    if (tid < 32) {
      if (tid < kbi) {
        const double cand = (bidx != INT64_MAX) ? pa[tid * rp + (int)(bidx - row0)] : 0.0;
        for (int rep = 0; rep < PX_RREPL; ++rep) ll_store(xw + px_row_at(buf, rep, b, 0, tid), (unsigned long long)__double_as_longlong(cand), epoch);
        if (b == 0) {
          const double cr = pa[tid * rp + (int)(col - row0)];
          for (int rep = 0; rep < PX_RREPL; ++rep) ll_store(xw + px_row_at(buf, rep, 0, 1, tid), (unsigned long long)__double_as_longlong(cr), epoch);
        }
      }
      if (tid < PX_HREPL) {
        unsigned long long* h = xw + px_hdr_at(buf, tid, b);
        ll_store(h, (unsigned long long)__double_as_longlong(best), epoch);
        ll_store(h + 2, (unsigned long long)bidx, epoch);
      }
    }
    // (c) poll the P headers, global arg-max (identical in every CTA), pivot bookkeeping
    double gb = -2.0;
    int64_t gi = INT64_MAX;
    if (tid < P) {
      const unsigned long long* h = xw + px_hdr_at(buf, b & (PX_HREPL - 1), tid);
      int fault = 0;
      gb = __longlong_as_double((long long)px_load(h, epoch, &fault));
      gi = (int64_t)px_load(h + 2, epoch, &fault);
      if (fault) fault_s = 1;
    }
    block_argmax(gb, gi, smax, sidx);
    if (tid == 0) {
      if (gi == INT64_MAX) gi = col;
      piv_s = gi;
      if (b == 0) ipiv[col] = gi + 1;
    }
    __syncthreads();
    const int64_t piv = piv_s;
    const bool own_piv = piv >= row0 && piv < row0 + nrows;
    const bool own_col = b == 0;
    // (d) the pivot row from its owner's message; complete the interchange
    if (tid < kbi) {
      int fault = 0;
      const int rep = b & (PX_RREPL - 1);
      const int owner = (int)((piv - c0) / rpc);
      const unsigned long long* src = (piv == col) ? xw + px_row_at(buf, rep, 0, 1, tid) : xw + px_row_at(buf, rep, owner, 0, tid);
      const double pv = __longlong_as_double((long long)px_load(src, epoch, &fault));
      urow[tid] = pv;
      if (own_piv && piv != col) {
        const double cr = __longlong_as_double((long long)px_load(xw + px_row_at(buf, rep, 0, 1, tid), epoch, &fault));
        pa[tid * rp + (int)(piv - row0)] = cr;
      }
      if (own_col) pa[tid * rp + (int)(col - row0)] = pv;
      if (fault) fault_s = 1;
    }
    __syncthreads();
    if (fault_s) {  // an exchange timed out: report through info and leave (every CTA times out on its own)
      if (b == 0 && tid == 0) *info = -1;
      break;
    }
    // (e) scale + rank-1 update of the rows below the diagonal
    const double pivval = urow[jj];
    if (pivval == 0.0) {
      if (b == 0 && tid == 0 && *info == 0) *info = (int)(col + 1);
    } else {
      const double inv = 1.0 / pivval;
      for (int r = tid; r < nrows; r += DT) {
        if (row0 + r > col) {
          const double l = pa[jj * rp + r] * inv;
          pa[jj * rp + r] = l;
          for (int c = jj + 1; c < kbi; ++c) pa[c * rp + r] = fma(-l, urow[c], pa[c * rp + r]);
        }
      }
    }
    __syncthreads();
  }
  for (int c = 0; c < kbi; ++c)
    for (int r = tid; r < nrows; r += DT) A[(c0 + c) * ld + row0 + r] = pa[c * rp + r];
}

// apply the interchanges ipiv[r0 .. r0+cnt) to columns [c_lo, c_hi) excluding [x_lo, x_hi)  (thread per column)
__global__ void __launch_bounds__(DT) swap_rows_kernel(double* __restrict__ A, int64_t ld, int64_t r0, int cnt, const int64_t* __restrict__ ipiv,
                                                        int64_t c_lo, int64_t c_hi, int64_t x_lo, int64_t x_hi) {
  int64_t c = c_lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= x_lo) c += (x_hi - x_lo);
  if (c >= c_hi) return;
  double* col = A + c * ld;
  for (int q = 0; q < cnt; ++q) {
    const int64_t r = r0 + q, p = ipiv[r] - 1;
    if (p != r) {
      const double t = col[r];
      col[r] = col[p];
      col[p] = t;
    }
  }
}

// U12 = L11^{-1} A12 for a whole outer panel in ONE launch: a CTA owns U12_NCB columns of A12 and keeps its kbo x U12_NCB tile in
// shared memory through all kbo / 32 block steps (warp-cooperative solve of the 32 x 32 unit-lower diagonal block — lanes are
// rows, the solved entries travel by shuffle — then the rows below are updated with the solved block read back as 16-byte
// broadcasts).  Replaces 31 dependent launches per outer step (16 solves of 32 rows + 15 updates), which had become pure launch
// latency even when A12 is thousands of columns wide.  FP64 FMA-bound: kbo^2 / 2 per column.  The inner panels use it too, with
// kbo = kbi <= 32: one block step and no rows below.
constexpr int U12_NCB = 16, U12_T = 256;
__global__ void __launch_bounds__(U12_T, 2) u12_fused_kernel(double* __restrict__ A, int64_t ld, int64_t k0, int kbo, int64_t k1, int64_t rest) {
  extern __shared__ double xs[];                 // [U12_NCB][kbo] column-major tile of A12
  __shared__ double Ld[NBI][NBI + 1];            // current diagonal block of L11 (strictly lower part used)
  __shared__ __align__(16) double xb[NBI][U12_NCB];  // the block just solved, row-major: one row = the 16 column values
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t c0 = k1 + (int64_t)blockIdx.x * U12_NCB;
  const int nc = (int)min((int64_t)U12_NCB, k1 + rest - c0);
  for (int idx = tid; idx < kbo * U12_NCB; idx += U12_T) {
    const int c = idx / kbo, r = idx - c * kbo;
    xs[idx] = (c < nc) ? A[(c0 + c) * ld + k0 + r] : 0.0;
  }
  __syncthreads();
  for (int b0 = 0; b0 < kbo; b0 += NBI) {
    const int kb = min(NBI, kbo - b0);
    for (int idx = tid; idx < kb * kb; idx += U12_T) {
      const int r = idx % kb, q = idx / kb;
      Ld[r][q] = A[(k0 + b0 + q) * ld + k0 + b0 + r];
    }
    __syncthreads();
    // ---- solve the diagonal block: warp w takes columns w, w + 8; lane = row; x_i is final after step i - 1
    for (int cc = warp; cc < U12_NCB; cc += U12_T / 32) {
      double x = (lane < kb) ? xs[cc * kbo + b0 + lane] : 0.0;
      for (int i = 0; i + 1 < kb; ++i) {
        const double xi = __shfl_sync(0xffffffffu, x, i);
        if (lane > i && lane < kb) x = fma(-Ld[lane][i], xi, x);
      }
      if (lane < kb) { xs[cc * kbo + b0 + lane] = x; xb[lane][cc] = x; }
    }
    __syncthreads();
    // ---- rows below the block: x[r, :] -= L[r, b0 : b0 + kb] * xb
    const int nb = kbo - b0 - kb;
    for (int r = tid; r < nb; r += U12_T) {
      const int rr = b0 + kb + r;
      double acc[U12_NCB];
#pragma unroll
      for (int c = 0; c < U12_NCB; ++c) acc[c] = xs[c * kbo + rr];
      const double* Lrow = A + (k0 + b0) * ld + k0 + rr;   // L[rr][b0 + q] = Lrow[q * ld]
      for (int q0 = 0; q0 < kb; q0 += 8) {
        double l[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) l[q] = (q0 + q < kb) ? Lrow[(int64_t)(q0 + q) * ld] : 0.0;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          if (q0 + q < kb) {
            const double2* xr = reinterpret_cast<const double2*>(xb[q0 + q]);
#pragma unroll
            for (int c = 0; c < U12_NCB; c += 2) {
              const double2 v = xr[c >> 1];
              acc[c] = fma(-l[q], v.x, acc[c]);
              acc[c + 1] = fma(-l[q], v.y, acc[c + 1]);
            }
          }
        }
      }
#pragma unroll
      for (int c = 0; c < U12_NCB; ++c) xs[c * kbo + rr] = acc[c];
    }
    __syncthreads();
  }
  for (int idx = tid; idx < kbo * U12_NCB; idx += U12_T) {
    const int c = idx / kbo, r = idx - c * kbo;
    if (c < nc) A[(c0 + c) * ld + k0 + r] = xs[idx];
  }
}

// ------------------------------------------------------------------ C -= A * B on the FP64 tensor cores
// A: M x K (lda), B: K x N (ldb), C: M x N (ldc), all column-major.  Shared-memory rows are padded by 4 doubles, so the
// fragment loads are bank-conflict free.
constexpr int GM_BM = 128, GM_BN = 64, GM_BK = 8, GM_PAD = 4, GM_STAGES = 4;
__device__ __forceinline__ void dmma_m8n8k4(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
// 8-byte asynchronous global->shared copy (LDGSTS); src_bytes = 0 zero-fills the destination (out-of-range elements)
__device__ __forceinline__ void cp_async8(double* smem_dst, const double* gsrc, int src_bytes) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n" ::"r"(d), "l"(gsrc), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// K is streamed in chunks of 8 through a 4-stage cp.async ring: three chunks are always in flight underneath the MMAs of the
// current one.  CTA = 8 warps (4 x 2), tile 128 (M) x 64 (N), each warp a 32 x 32 sub-tile = 4 x 4 DMMA m8n8k4 accumulator
// fragments (64 registers): 118 registers per thread -> two CTAs = 16 warps per SM.  The FP64 tensor pipe of this part is fed
// by warps, not by tile size: fewer warps per SM (4 warps x (32 x 64) per CTA, or a persistent 128 x 128-tile kernel with ONE
// 8-warp CTA per SM despite its better arithmetic intensity) factor the matrix more slowly.
constexpr int G8_T = 256;
constexpr int GM_SWZ = 16;  // tile columns per rasterisation group
__global__ void __launch_bounds__(G8_T, 2) gemm_sub_w8_kernel(int64_t M, int64_t N, int K, const double* __restrict__ A, int64_t lda,
                                                               const double* __restrict__ B, int64_t ldb, double* __restrict__ C, int64_t ldc) {
  extern __shared__ double gsm[];
  double(*As)[GM_BK][GM_BM + GM_PAD] = reinterpret_cast<double(*)[GM_BK][GM_BM + GM_PAD]>(gsm);
  double(*Bs)[GM_BK][GM_BN + GM_PAD] = reinterpret_cast<double(*)[GM_BK][GM_BN + GM_PAD]>(gsm + GM_STAGES * GM_BK * (GM_BM + GM_PAD));
  // Tile order: CTAs are dispatched with blockIdx.x fastest; taken literally every tile column (blockIdx.y) streams the whole
  // A panel (M x K: 132 MB at n = 32768, K = 512 — more than the 50 MB L2 keeps) from DRAM again, tens of GB of DRAM reads for
  // one trailing update.  Remapped in groups of GM_SWZ tile columns: consecutive CTAs
  // share one A tile and cycle through the group's B tiles (4 MB, L2-resident), so A is read once per group.
  int tile_m = blockIdx.x, tile_n = blockIdx.y;
  {
    const int tm = gridDim.x, tn = gridDim.y;
    const int64_t lin = (int64_t)blockIdx.y * tm + blockIdx.x, per_group = (int64_t)GM_SWZ * tm;
    const int grp = (int)(lin / per_group), first_n = grp * GM_SWZ;
    const int gsz = min(GM_SWZ, tn - first_n);
    const int r = (int)(lin - (int64_t)grp * per_group);
    tile_m = r / gsz;
    tile_n = first_n + (r - tile_m * gsz);
  }
  const int64_t m0 = (int64_t)tile_m * GM_BM, n0 = (int64_t)tile_n * GM_BN;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = (warp & 3) * 32, wn = (warp >> 2) * 32;
  const int g = lane >> 2, t4 = lane & 3;
  const int am = tid & 127, ak = tid >> 7;             // A staging: thread covers k = ak + 2 q, q = 0 .. GM_BK/2-1
  const int bk = tid & (GM_BK - 1), bn = tid / GM_BK;  // B staging: thread covers n = bn + (256/GM_BK) q, q = 0 .. GM_BK/4-1
  const bool m_ok = m0 + am < M;
  const double* a_src = A + (m_ok ? m0 + am : 0);
  auto issue_chunk = [&](int ch) {
    const int st = ch % GM_STAGES, kc = ch * GM_BK;
#pragma unroll
    for (int q = 0; q < GM_BK / 2; ++q) {
      const int k = ak + 2 * q;
      const bool ok = m_ok && (kc + k < K);
      cp_async8(&As[st][k][am], a_src + (int64_t)(ok ? kc + k : 0) * lda, ok ? 8 : 0);
    }
#pragma unroll
    for (int q = 0; q < GM_BK / 4; ++q) {
      const int64_t nn = n0 + bn + (G8_T / GM_BK) * q;
      const bool ok = (nn < N) && (kc + bk < K);
      cp_async8(&Bs[st][bk][bn + (G8_T / GM_BK) * q], B + (ok ? nn * ldb + kc + bk : 0), ok ? 8 : 0);
    }
  };
  double acc[4][4][2];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b][0] = acc[a][b][1] = 0.0;
  const int nchunks = (K + GM_BK - 1) / GM_BK;
#pragma unroll
  for (int s = 0; s < GM_STAGES - 1; ++s) {
    if (s < nchunks) issue_chunk(s);
    cp_async_commit();
  }
  for (int ch = 0; ch < nchunks; ++ch) {
    cp_async_wait<GM_STAGES - 2>();
    __syncthreads();
    if (ch + GM_STAGES - 1 < nchunks) issue_chunk(ch + GM_STAGES - 1);
    cp_async_commit();
    const int st = ch % GM_STAGES;
#pragma unroll
    for (int kk = 0; kk < GM_BK; kk += 4) {
      double af[4], bf[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) af[a] = As[st][kk + t4][wm + a * 8 + g];
#pragma unroll
      for (int b = 0; b < 4; ++b) bf[b] = Bs[st][kk + t4][wn + b * 8 + g];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) dmma_m8n8k4(acc[a][b][0], acc[a][b][1], af[a], bf[b]);
    }
  }
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int64_t i = m0 + wm + a * 8 + g;
      const int64_t j = n0 + wn + b * 8 + 2 * t4;
      if (i < M) {
        if (j < N) C[j * ldc + i] -= acc[a][b][0];
        if (j + 1 < N) C[(j + 1) * ldc + i] -= acc[a][b][1];
      }
    }
}

constexpr size_t GEMM_SMEM = sizeof(double) * GM_STAGES * GM_BK * ((GM_BM + GM_PAD) + (GM_BN + GM_PAD));

int32_t gemm_sub(b200_ctx* ctx, int64_t M, int64_t N, int K, const double* A, int64_t lda, const double* B, int64_t ldb, double* C, int64_t ldc) {
  if (M <= 0 || N <= 0 || K <= 0) return B200_OK;
  dim3 grid((unsigned)((M + GM_BM - 1) / GM_BM), (unsigned)((N + GM_BN - 1) / GM_BN));
  PLAUNCH(ctx, B200_KID_LU_GEMM, 2.0 * (double)M * (double)N * (double)K /* flops, not bytes */, gemm_sub_w8_kernel, grid, G8_T, GEMM_SMEM, M, N, K, A,
          lda, B, ldb, C, ldc);
  return B200_OK;
}

// ------------------------------------------------------------------ triangular solves (nrhs small)
__global__ void __launch_bounds__(DT) apply_pivots_kernel(int64_t n, int64_t nrhs, const int64_t* __restrict__ ipiv, double* __restrict__ B, int64_t ldb) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= nrhs) return;
  double* b = B + r * ldb;
  for (int64_t k = 0; k < n; ++k) {
    const int64_t p = ipiv[k] - 1;
    if (p != k) { const double t = b[k]; b[k] = b[p]; b[p] = t; }
  }
}
// one block step of the forward (unit lower) or backward (upper) substitution: solve the NBI x NBI diagonal block, then
// subtract its contribution from the rest of the right-hand side (all CTAs).
__global__ void __launch_bounds__(64) trisolve_diag_kernel(int lower, const double* __restrict__ A, int64_t ld, int64_t k0, int kb, double* __restrict__ b) {
  __shared__ double T[NBI][NBI + 1];
  __shared__ double x[NBI];
  for (int t = threadIdx.x; t < kb * kb; t += blockDim.x) {
    const int r = t % kb, c = t / kb;
    T[r][c] = A[(k0 + c) * ld + k0 + r];
  }
  for (int t = threadIdx.x; t < kb; t += blockDim.x) x[t] = b[k0 + t];
  __syncthreads();
  if (threadIdx.x == 0) {
    if (lower) {
      for (int r = 0; r < kb; ++r) { double s = x[r]; for (int q = 0; q < r; ++q) s -= T[r][q] * x[q]; x[r] = s; }
    } else {
      for (int r = kb - 1; r >= 0; --r) { double s = x[r]; for (int q = r + 1; q < kb; ++q) s -= T[r][q] * x[q]; x[r] = s / T[r][r]; }
    }
  }
  __syncthreads();
  for (int t = threadIdx.x; t < kb; t += blockDim.x) b[k0 + t] = x[t];
}
__global__ void __launch_bounds__(DT) trisolve_update_kernel(int lower, int64_t n, const double* __restrict__ A, int64_t ld, int64_t k0, int kb,
                                                              double* __restrict__ b) {
  __shared__ double x[NBI];
  for (int t = threadIdx.x; t < kb; t += blockDim.x) x[t] = b[k0 + t];
  __syncthreads();
  const int64_t lo = lower ? k0 + kb : 0, hi = lower ? n : k0;
  const int64_t i = lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= hi) return;
  double s = b[i];
  for (int q = 0; q < kb; ++q) s = fma(-A[(k0 + q) * ld + i], x[q], s);
  b[i] = s;
}
}  // namespace

namespace {
// ---- Levenberg-Marquardt normal form (levenberg_marquardt.jl / damped_newton.jl :normal_form): C = J' J, and the diagonal of it
// C[i, j] = sum_k J[k, i] J[k, j]: both operands are contiguous in k (column-major J), 64 x 64 output tile per CTA, 16 x 16
// threads with a 4 x 4 register block each.  CUDA-core FP64: LM serves small dense systems, this is not a roofline kernel.
constexpr int LMT = 64, LMK = 16;
__global__ void __launch_bounds__(256) gram_kernel(int64_t n, const double* __restrict__ J, int64_t ld, double* __restrict__ C, int64_t ldc) {
  __shared__ double Ai[LMK][LMT + 1], Aj[LMK][LMT + 1];
  const int64_t i0 = (int64_t)blockIdx.x * LMT, j0 = (int64_t)blockIdx.y * LMT;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  double acc[4][4] = {};
  for (int64_t k0 = 0; k0 < n; k0 += LMK) {
    for (int e = threadIdx.x; e < LMK * LMT; e += 256) {
      const int k = e % LMK, c = e / LMK;   // k fastest: coalesced down the column
      const int64_t gk = k0 + k;
      Ai[k][c] = (gk < n && i0 + c < n) ? J[(i0 + c) * ld + gk] : 0.0;
      Aj[k][c] = (gk < n && j0 + c < n) ? J[(j0 + c) * ld + gk] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < LMK; ++k) {
      double a[4], b[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) { a[q] = Ai[k][tx + 16 * q]; b[q] = Aj[k][ty + 16 * q]; }
#pragma unroll
      for (int p = 0; p < 4; ++p)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[p][q] = fma(a[p], b[q], acc[p][q]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int64_t i = i0 + tx + 16 * p, j = j0 + ty + 16 * q;
      if (i < n && j < n) C[j * ldc + i] = acc[p][q];
    }
}
// dtd[j] = max(dtd[j], C[j, j])  (update_levenberg_marquardt_diagonal!!) ; C[j, j] += lambda * dtd[j]  (dampen_jacobian!!)
__global__ void __launch_bounds__(256) lm_damp_kernel(int64_t n, double* __restrict__ C, int64_t ldc, double* __restrict__ dtd, double lambda) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const double d = fmax(dtd[j], C[j * ldc + j]);
  dtd[j] = d;
  C[j * ldc + j] += lambda * d;
}
}  // namespace
namespace {
// ---- Rescue of a singular LU (SURVEY.md §8a a5; the reference's default dense solver falls back from a failed LU to a
// column-pivoted QR, lib/NonlinearSolveBase/src/linear_solve.jl:48-55, ext/NonlinearSolveBaseLinearSolveExt.jl:42-49).
// Householder QR with column pivoting, unblocked, ONE persistent CTA (32 warps, a warp per trailing column, coalesced down the
// column): a rescue path for the small dense systems where a singular Jacobian can be met, not a roofline kernel.
// On exit: R in the upper triangle, the Householder vectors below the diagonal (v_k = 1 implied), tau, jpvt, and the numerical
// rank (|R_kk| > n eps |R_00|).
constexpr int QR_T = 1024;
__global__ void __launch_bounds__(QR_T, 1) qrcp_kernel(int64_t n, double* __restrict__ A, int64_t ld, double* __restrict__ tau, int32_t* __restrict__ jpvt,
                                                        double* __restrict__ colnorm, int32_t* __restrict__ rank_out) {
  __shared__ double red_v[32];
  __shared__ int64_t red_i[32];
  __shared__ double s_a, s_b;
  __shared__ int s_p;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int64_t j = tid; j < n; j += QR_T) jpvt[j] = (int32_t)j;
  __syncthreads();
  double r00 = 0.0;
  int rank = 0;
  for (int64_t k = 0; k < n; ++k) {
    // squared norms of the trailing parts of columns k .. n-1 (recomputed: downdating loses accuracy exactly where it matters)
    for (int64_t j = k + warp; j < n; j += 32) {
      const double* c = A + j * ld;
      double s = 0.0;
      for (int64_t i = k + lane; i < n; i += 32) s = fma(c[i], c[i], s);
      s = warp_sum(s);
      if (lane == 0) colnorm[j] = s;
    }
    __syncthreads();
    double best = -1.0;
    int64_t bi = k;
    for (int64_t j = k + tid; j < n; j += QR_T) { const double v = colnorm[j]; if (v > best) { best = v; bi = j; } }
    block_argmax(best, bi, red_v, red_i);  // result in warp 0
    if (tid == 0) { s_p = (int)bi; s_a = best; }
    __syncthreads();
    const int64_t p = s_p;
    const double cn2 = s_a;
    if (p != k) {  // swap columns k and p (all rows) and the permutation
      double *ck = A + k * ld, *cp = A + p * ld;
      for (int64_t i = tid; i < n; i += QR_T) { const double t = ck[i]; ck[i] = cp[i]; cp[i] = t; }
      if (tid == 0) { const int32_t t = jpvt[k]; jpvt[k] = jpvt[p]; jpvt[p] = t; }
    }
    __syncthreads();
    // Householder reflector of column k: H = I - tau v v', v = (1, A[k+1:, k] / (alpha - beta)), H x = beta e_1
    double* ck = A + k * ld;
    if (tid == 0) {
      const double alpha = ck[k];
      const double xn2 = fmax(cn2 - alpha * alpha, 0.0);
      double beta = 0.0, t = 0.0, scal = 0.0;
      if (xn2 > 0.0 || alpha != 0.0) {
        beta = -copysign(sqrt(alpha * alpha + xn2), alpha);
        t = (beta - alpha) / beta;
        scal = (xn2 > 0.0) ? 1.0 / (alpha - beta) : 0.0;
        if (xn2 == 0.0) { beta = alpha; t = 0.0; }
      }
      ck[k] = beta;
      tau[k] = t;
      s_a = t; s_b = scal;
    }
    __syncthreads();
    const double t = s_a, scal = s_b;
    for (int64_t i = k + 1 + tid; i < n; i += QR_T) ck[i] *= scal;
    __syncthreads();
    if (k == 0) r00 = fabs(ck[0]);
    if (fabs(ck[k]) > (double)n * 2.220446049250313e-16 * r00) rank = (int)k + 1;
    // apply H to the trailing columns: w = v' a_j ; a_j -= tau w v     (a warp per column)
    if (t != 0.0)
      for (int64_t j = k + 1 + warp; j < n; j += 32) {
        double* c = A + j * ld;
        double s = (lane == 0) ? c[k] : 0.0;
        for (int64_t i = k + 1 + lane; i < n; i += 32) s = fma(ck[i], c[i], s);
        s = warp_sum(s) * t;
        if (lane == 0) c[k] -= s;
        for (int64_t i = k + 1 + lane; i < n; i += 32) c[i] = fma(-s, ck[i], c[i]);
      }
    __syncthreads();
  }
  if (tid == 0) *rank_out = rank;
}
// x = P [R11^-1 (Q' b)(1:r) ; 0]  — the basic least-squares solution of the rank-r system; b is overwritten
__global__ void __launch_bounds__(QR_T, 1) qrcp_solve_kernel(int64_t n, const double* __restrict__ A, int64_t ld, const double* __restrict__ tau,
                                                              const int32_t* __restrict__ jpvt, const int32_t* __restrict__ rank_in, double* __restrict__ b,
                                                              double* __restrict__ x) {
  __shared__ double red[32];
  __shared__ double s_s;
  const int tid = threadIdx.x;
  const int r = *rank_in;
  for (int64_t k = 0; k < n; ++k) {  // c = Q' b: reflectors in order
    const double* ck = A + k * ld;
    double s = 0.0;
    for (int64_t i = k + 1 + tid; i < n; i += QR_T) s = fma(ck[i], b[i], s);
    s = block_sum(s, red);
    if (tid == 0) { s_s = (s + b[k]) * tau[k]; b[k] -= s_s; }
    __syncthreads();
    const double ss = s_s;
    for (int64_t i = k + 1 + tid; i < n; i += QR_T) b[i] = fma(-ss, ck[i], b[i]);
    __syncthreads();
  }
  for (int64_t k = r - 1; k >= 0; --k) {  // R11 y = c(1:r), column-oriented back substitution in place
    const double* ck = A + k * ld;
    if (tid == 0) { s_s = b[k] / ck[k]; b[k] = s_s; }
    __syncthreads();
    const double yk = s_s;
    for (int64_t i = tid; i < k; i += QR_T) b[i] = fma(-ck[i], yk, b[i]);
    __syncthreads();
  }
  for (int64_t k = tid; k < n; k += QR_T) x[jpvt[k]] = (k < r) ? b[k] : 0.0;
}
}  // namespace
int32_t b200i_qrcp_solve(b200_ctx* ctx, int64_t n, double* A, int64_t ld, double* b, double* x, double* work /* >= 2 n doubles */, int32_t* jpvt_dev /* n + 1 */,
                         int32_t* rank_host) {
  double* tau = work;
  double* colnorm = work + n;
  LAUNCH(ctx, qrcp_kernel, 1, QR_T, 0, n, A, ld, tau, jpvt_dev, colnorm, jpvt_dev + n);
  LAUNCH(ctx, qrcp_solve_kernel, 1, QR_T, 0, n, (const double*)A, ld, (const double*)tau, (const int32_t*)jpvt_dev, (const int32_t*)(jpvt_dev + n), b, x);
  CHECK_LAUNCH(ctx);
  if (rank_host) {
    CUDA_TRY(ctx, cudaMemcpyAsync(rank_host, jpvt_dev + n, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  }
  return B200_OK;
}

int32_t b200i_gram(b200_ctx* ctx, int64_t n, const double* J, int64_t ld, double* C, int64_t ldc) {
  dim3 grid((unsigned)((n + LMT - 1) / LMT), (unsigned)((n + LMT - 1) / LMT));
  LAUNCH(ctx, gram_kernel, grid, 256, 0, n, J, ld, C, ldc);
  CHECK_LAUNCH(ctx);
  return B200_OK;
}
int32_t b200i_lm_damp(b200_ctx* ctx, int64_t n, double* C, int64_t ldc, double* dtd, double lambda) {
  LAUNCH(ctx, lm_damp_kernel, (int)((n + 255) / 256), 256, 0, n, C, ldc, dtd, lambda);
  CHECK_LAUNCH(ctx);
  return B200_OK;
}

namespace {
__global__ void __launch_bounds__(256) diag_shift_kernel(int64_t n, double* __restrict__ A, int64_t ld, double shift) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) A[i * ld + i] += shift;
}
}  // namespace
namespace {
// ---- quasi-Newton (Broyden) level-2 kernels on the stored inverse: HBM-bound, one pass over the n x n matrix each
// A[:, j] += c * w[j] for a tile of columns: 16-byte accesses down the column, c kept in registers across GER_CPB columns
constexpr int GER_T = 256, GER_CPB = 8;
__global__ void __launch_bounds__(GER_T) ger_kernel(int64_t n, double* __restrict__ A, int64_t ld, const double* __restrict__ c, const double* __restrict__ w) {
  const int64_t i = ((int64_t)blockIdx.x * GER_T + threadIdx.x) * 2;
  const int64_t j0 = (int64_t)blockIdx.y * GER_CPB;
  if (i >= n) return;
  const bool pair = (i + 1 < n) && ((ld & 1) == 0);
  const double c0 = c[i], c1 = (i + 1 < n) ? c[i + 1] : 0.0;
#pragma unroll
  for (int jj = 0; jj < GER_CPB; ++jj) {
    const int64_t j = j0 + jj;
    if (j >= n) break;
    const double wj = w[j];
    double* col = A + j * ld + i;
    if (pair) {
      double2 a = *reinterpret_cast<double2*>(col);
      a.x = fma(c0, wj, a.x); a.y = fma(c1, wj, a.y);
      *reinterpret_cast<double2*>(col) = a;
    } else {
      col[0] = fma(c0, wj, col[0]);
      if (i + 1 < n) col[1] = fma(c1, wj, col[1]);
    }
  }
}
__global__ void __launch_bounds__(256) scaled_identity_kernel(int64_t n, double* __restrict__ A, int64_t ld, double d) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t j = blockIdx.y;
  if (i < n) A[j * ld + i] = (i == j) ? d : 0.0;
}
}  // namespace
namespace {
// Klement with a diagonal approximate Jacobian: everything is elementwise
__global__ void __launch_bounds__(256) klement_descent_kernel(int64_t n, const double* __restrict__ J, const double* __restrict__ fu, double* __restrict__ du) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) du[i] = -(fu[i] / J[i]);   // J \ fu for a Diagonal, then @. du *= -1
}
__global__ void __launch_bounds__(256) klement_update_kernel(int64_t n, double* __restrict__ J, const double* __restrict__ fu, double* __restrict__ fu_cache,
                                                             const double* __restrict__ du) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double j = J[i], d = du[i], f = fu[i];
  // The numerator f - f_prev - J du cancels to rounding level near the root and is then divided by J^2 du^2 ~ 1e-15: the rule is
  // ill-conditioned there, and a fused multiply-add in it sends the iteration somewhere else than the reference's unfused
  // broadcast does (observed: blow-up at the step where the reference converges).  Every operation is therefore rounded
  // separately, in the broadcast's order:  J += (((f - f_prev) - J du) / D) * du * J^2,  D = J^2 du^2 (1e-5 when zero).
  const double jj = __dmul_rn(j, j);
  const double jdu = __dmul_rn(jj, __dmul_rn(d, d));
  const double num = __dadd_rn(__dadd_rn(f, -fu_cache[i]), -__dmul_rn(j, d));
  const double t = __dmul_rn(__dmul_rn(__ddiv_rn(num, jdu == 0.0 ? 1.0e-5 : jdu), d), jj);
  J[i] = __dadd_rn(j, t);
  fu_cache[i] = f;
}
}  // namespace
int32_t b200i_klement_descent(b200_ctx* ctx, int64_t n, const double* J, const double* fu, double* du) {
  LAUNCH(ctx, klement_descent_kernel, (int)((n + 255) / 256), 256, 0, n, J, fu, du);
  CHECK_LAUNCH(ctx);
  return B200_OK;
}
int32_t b200i_klement_update(b200_ctx* ctx, int64_t n, double* J, const double* fu, double* fu_cache, const double* du) {
  LAUNCH(ctx, klement_update_kernel, (int)((n + 255) / 256), 256, 0, n, J, fu, fu_cache, du);
  CHECK_LAUNCH(ctx);
  return B200_OK;
}
int32_t b200i_ger(b200_ctx* ctx, int64_t n, double* A, int64_t ld, const double* c, const double* w) {
  const dim3 grid((unsigned)((n + 2 * GER_T - 1) / (2 * GER_T)), (unsigned)((n + GER_CPB - 1) / GER_CPB));
  LAUNCH(ctx, ger_kernel, grid, GER_T, 0, n, A, ld, c, w);
  CHECK_LAUNCH(ctx);
  return B200_OK;
}
int32_t b200i_scaled_identity(b200_ctx* ctx, int64_t n, double* A, int64_t ld, double d) {
  const dim3 grid((unsigned)((n + 255) / 256), (unsigned)n);
  LAUNCH(ctx, scaled_identity_kernel, grid, 256, 0, n, A, ld, d);
  CHECK_LAUNCH(ctx);
  return B200_OK;
}
int32_t b200i_diag_shift(b200_ctx* ctx, int64_t n, double* A, int64_t ld, double shift) {
  LAUNCH(ctx, diag_shift_kernel, (int)((n + 255) / 256), 256, 0, n, A, ld, shift);
  CHECK_LAUNCH(ctx);
  return B200_OK;
}

extern "C" {
int32_t b200_dense_jac_fill(b200_problem* p, const double* u, double* J, int64_t ld) {
  B200_DEVICE_GUARD(p ? p->ctx : nullptr);
  b200_ctx* ctx = p->ctx;
  const int64_t n = p->n;
  B200_REQUIRE(ctx, ld >= n, "dense_jac_fill: ld < n");
  if (p->jac_dense_cb) {  // jac!(J, u, p)   jacobian.jl:241-243
    B200_REQUIRE(ctx, ld == n, "dense_jac_fill: a user jac! fills a contiguous n x n matrix (ld must equal n)");
    B200_TRY(b200i_sync_for_callback(ctx));
    return p->jac_dense_cb(p->user, u, J) == 0 ? B200_OK : ctx->fail(B200_ERR_CALLBACK, "jac! callback failed", __FILE__, __LINE__);
  }
  if (p->kind != B200_PROB_CALLBACK) CUDA_TRY(ctx, cudaMemsetAsync(J, 0, sizeof(double) * ld * n, ctx->stream));
  const int grid = (int)((n + DT - 1) / DT);
  switch (p->kind) {
    case B200_PROB_BRUSS2D:
    case B200_PROB_BRUSS3D:
      PLAUNCH(ctx, B200_KID_LU_OTHER, 8.0 * (double)ld * (double)n, bruss_dense_fill_kernel, grid, DT, 0, p->kind == B200_PROB_BRUSS2D ? 2 : 3, p->N, p->a, p->A,
              u, J, ld);
      break;
    case B200_PROB_QUADRATIC:
    case B200_PROB_TRIDIAG_QUAD:
      LAUNCH(ctx, small_dense_fill_kernel, grid, DT, 0, p->kind == B200_PROB_QUADRATIC ? 0 : 1, n, u, J, ld);
      break;
    case B200_PROB_CALLBACK: {  // n operator applications on unit vectors (what chunk-1 forward AD would do)
      double* e = nullptr;
      CUDA_TRY(ctx, cudaMalloc(&e, sizeof(double) * n));
      for (int64_t j = 0; j < n; ++j) {
        LAUNCH(ctx, unit_vector_kernel, grid, DT, 0, n, j, e);
        int32_t s = b200_jvp(p, u, e, J + j * ld);
        if (s != B200_OK) { cudaFree(e); return s; }
      }
      cudaStreamSynchronize(ctx->stream);
      cudaFree(e);
    } break;
    default: return ctx->fail(B200_ERR_INVALID, "unknown problem kind", __FILE__, __LINE__);
  }
  CHECK_LAUNCH(ctx);
  return B200_OK;
}

int32_t b200_getrf(b200_ctx* ctx, int64_t n, double* A, int64_t ld, int64_t* ipiv, int32_t* info_host) {
  B200_DEVICE_GUARD(ctx);
  B200_REQUIRE(ctx, n > 0 && ld >= n, "getrf: bad dimensions");
  int* info = reinterpret_cast<int*>(ctx->d_partials + 2 * B200_RED_MAX_BLOCKS);  // first zero pivot (col + 1), -1: timeout
  CUDA_TRY(ctx, cudaMemsetAsync(info, 0, sizeof(int), ctx->stream));
  if (!ctx->d_lu_xchg && cudaMalloc(&ctx->d_lu_xchg, sizeof(unsigned long long) * PX_WORDS) != cudaSuccess) {
    cudaGetLastError();
    return ctx->fail(B200_ERR_NOMEM, "getrf: exchange tables", __FILE__, __LINE__);
  }
  CUDA_TRY(ctx, cudaMemsetAsync(ctx->d_lu_xchg, 0, sizeof(unsigned long long) * PX_WORDS, ctx->stream));  // epochs are column numbers: valid for one factorisation
  CUDA_TRY(ctx, cudaFuncSetAttribute(panel_coop_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
  CUDA_TRY(ctx, cudaFuncSetAttribute(gemm_sub_w8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GEMM_SMEM));
  CUDA_TRY(ctx, cudaFuncSetAttribute(u12_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(double) * 512 * U12_NCB)));
  if (!ctx->aux_stream) {
    // highest priority: while the trailing update's CTAs drain and refill, the block scheduler hands freed SM slots to the
    // look-ahead panel first, so the (latency-bound, cooperative) panel runs underneath the GEMM instead of after it
    int prio_lo = 0, prio_hi = 0;
    CUDA_TRY(ctx, cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
    CUDA_TRY(ctx, cudaStreamCreateWithPriority(&ctx->aux_stream, cudaStreamNonBlocking, prio_hi));
    CUDA_TRY(ctx, cudaEventCreateWithFlags(&ctx->ev_a, cudaEventDisableTiming));
    CUDA_TRY(ctx, cudaEventCreateWithFlags(&ctx->ev_b, cudaEventDisableTiming));
  }
  cudaStream_t s_main = ctx->stream, s_panel = ctx->aux_stream;

  // factor the outer panel A[k0:n, k0:k0+kbo] (inner panels of NBI columns); issued on whatever ctx->stream currently is
  auto factor_panel = [&](int64_t k0, int kbo) -> int32_t {
    const int64_t k1 = k0 + kbo;
    for (int i0 = 0; i0 < kbo; i0 += NBI) {
      const int kbi = std::min(NBI, kbo - i0);
      const int64_t c0 = k0 + i0, c1 = c0 + kbi;
      {
        // cooperative panel: as many CTAs as keep >= 128 rows each, at most one per SM (all co-resident)
        const int64_t m = n - c0;
        // (capping the panel below one CTA per SM to leave SMs to the concurrent trailing update does not help)
        int P = (int)std::min<int64_t>(std::min(ctx->sm_count, PS_MAX), std::max<int64_t>(1, (m + 127) / 128));
        int rpc = (int)((m + P - 1) / P);
        P = (int)((m + rpc - 1) / rpc);
        const size_t smem = sizeof(double) * (size_t)kbi * (size_t)(rpc | 1);
        B200_TRY(coop_launch(ctx, B200_KID_LU_PANEL, 0.0, panel_coop_kernel, P, DT, smem, n, A, ld, c0, kbi, rpc, ipiv, info, ctx->d_lu_xchg));
        // the panel's interchanges applied to the other columns of the outer panel
        if (kbo - kbi > 0)
          PLAUNCH(ctx, B200_KID_LU_OTHER, 0.0, swap_rows_kernel, (int)((kbo - kbi + DT - 1) / DT), DT, 0, A, ld, c0, kbi, (const int64_t*)ipiv, k0, k1, c0, c1);
      }
      const int64_t rest = k1 - c1;  // rest of the outer panel: U = L11^{-1} A12 ; A22 -= L21 U
      if (rest > 0) {
        PLAUNCH(ctx, B200_KID_LU_OTHER, 0.0, u12_fused_kernel, (int)((rest + U12_NCB - 1) / U12_NCB), U12_T, sizeof(double) * kbi * U12_NCB, A, ld, c0,
                kbi, c1, rest);
        B200_TRY(gemm_sub(ctx, n - c1, rest, kbi, A + c0 * ld + c1, ld, A + c1 * ld + c0, ld, A + c1 * ld + c1, ld));
      }
    }
    return B200_OK;
  };

  // outer block (the K of the trailing update): 512 for the big factorisations halves the C read-modify-write traffic
  // (n = 32768: 1.08 s -> 1.02 s; 768 buys nothing more), 256 below
  const int NBO = n >= 16384 ? 512 : NBO_DEFAULT;  // A/B knob for the outer block
  B200_TRY(factor_panel(0, (int)std::min<int64_t>(NBO, n)));
  for (int64_t k0 = 0; k0 < n; k0 += NBO) {
    const int kbo = (int)std::min<int64_t>(NBO, n - k0);
    const int64_t k1 = k0 + kbo;
    // ---- interchanges of this panel applied to the columns left and right of it
    if (n - kbo > 0)
      PLAUNCH(ctx, B200_KID_LU_OTHER, 0.0, swap_rows_kernel, (int)((n - kbo + DT - 1) / DT), DT, 0, A, ld, k0, kbo, (const int64_t*)ipiv, (int64_t)0, n, k0, k1);
    const int64_t rest = n - k1;
    if (rest <= 0) break;
    // ---- U12 = L11^{-1} A12: one fused launch (column blocks of 16 stay in shared memory through all 16 block steps)
    {
      const size_t smem = sizeof(double) * (size_t)kbo * U12_NCB;
      PLAUNCH(ctx, B200_KID_LU_OTHER, 0.0, u12_fused_kernel, (int)((rest + U12_NCB - 1) / U12_NCB), U12_T, smem, A, ld, k0, kbo, k1, rest);
    }
    // ---- trailing update on the FP64 tensor cores, with look-ahead: first the columns of the NEXT panel, whose
    //      factorisation (latency-bound, few SMs) then runs on a second stream underneath the rest of the GEMM.
    const int kbn = (int)std::min<int64_t>(NBO, rest);
    B200_TRY(gemm_sub(ctx, rest, kbn, kbo, A + k0 * ld + k1, ld, A + k1 * ld + k0, ld, A + k1 * ld + k1, ld));
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_a, s_main));
    CUDA_TRY(ctx, cudaStreamWaitEvent(s_panel, ctx->ev_a, 0));
    ctx->stream = s_panel;
    int32_t st = factor_panel(k1, kbn);
    ctx->stream = s_main;
    B200_TRY(st);
    CUDA_TRY(ctx, cudaEventRecord(ctx->ev_b, s_panel));
    if (rest - kbn > 0)
      B200_TRY(gemm_sub(ctx, rest, rest - kbn, kbo, A + k0 * ld + k1, ld, A + (k1 + kbn) * ld + k0, ld, A + (k1 + kbn) * ld + k1, ld));
    CUDA_TRY(ctx, cudaStreamWaitEvent(s_main, ctx->ev_b, 0));
  }
  CHECK_LAUNCH(ctx);
  if (info_host) {
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->h_scalars + 16, info, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    *info_host = *reinterpret_cast<int*>(ctx->h_scalars + 16);
    if (*info_host < 0) return ctx->fail(B200_ERR_CUDA, "getrf: the panel's cross-CTA exchange timed out", __FILE__, __LINE__);
  }
  return B200_OK;
}

int32_t b200_getrs(b200_ctx* ctx, int64_t n, int64_t nrhs, const double* A, int64_t ld, const int64_t* ipiv, double* B, int64_t ldb) {
  B200_DEVICE_GUARD(ctx);
  B200_REQUIRE(ctx, n > 0 && nrhs > 0 && ld >= n && ldb >= n, "getrs: bad dimensions");
  LAUNCH(ctx, apply_pivots_kernel, (int)((nrhs + DT - 1) / DT), DT, 0, n, nrhs, ipiv, B, ldb);
  for (int64_t r = 0; r < nrhs; ++r) {
    double* b = B + r * ldb;
    for (int64_t k0 = 0; k0 < n; k0 += NBI) {  // L y = P b
      const int kb = (int)std::min<int64_t>(NBI, n - k0);
      LAUNCH(ctx, trisolve_diag_kernel, 1, 64, 0, 1, A, ld, k0, kb, b);
      const int64_t rest = n - (k0 + kb);
      if (rest > 0) LAUNCH(ctx, trisolve_update_kernel, (int)((rest + DT - 1) / DT), DT, 0, 1, n, A, ld, k0, kb, b);
    }
    const int64_t nblk = (n + NBI - 1) / NBI;
    for (int64_t blk = nblk - 1; blk >= 0; --blk) {  // U x = y
      const int64_t k0 = blk * NBI;
      const int kb = (int)std::min<int64_t>(NBI, n - k0);
      LAUNCH(ctx, trisolve_diag_kernel, 1, 64, 0, 0, A, ld, k0, kb, b);
      if (k0 > 0) LAUNCH(ctx, trisolve_update_kernel, (int)((k0 + DT - 1) / DT), DT, 0, 0, n, A, ld, k0, kb, b);
    }
  }
  CHECK_LAUNCH(ctx);
  return B200_OK;
}
}  // extern "C"
