// gmres.cu — device-resident GMRES (SURVEY.md §8a row a3, kernels K3/K4), multi-kernel engine.
//
// Replaces what the reference reaches through `solve!(cache.lincache)` at
// lib/NonlinearSolveBase/ext/NonlinearSolveBaseLinearSolveExt.jl:26 (LinearSolve.KrylovJL_GMRES -> Krylov.gmres!):
// Arnoldi + Gram-Schmidt + Givens reflections, stop at ||r|| <= atol + rtol ||r0||, no restart by default.
//
// Design: the Krylov basis, the Hessenberg/Givens recurrence, the residual estimate and the stopping decision
// all live on the device.  An Arnoldi iteration is a fixed sequence of kernels with no host round trip
// (operator apply -> multi-dot -> update+norm -> givens -> normalise); the host only polls a status word every
// `check_every` iterations, and kernels enqueued after convergence early-exit on that word.
//   multi-dot   h = V_k' w   : every CTA owns a contiguous row range, streams JT basis columns at a time with 16-byte
//                              loads, warp-shuffle + shared-memory block reduction, per-CTA partials summed in fixed
//                              order (deterministic, no atomics)
//   update      w -= V_k h   : one pass over the basis with the ||w||^2 partial fused into the epilogue
//   MGS (reference-parity mode): per basis vector one fused pass  w -= h_i v_i ; h_{i+1} = v_{i+1}.w
// Orthogonalisation modes: MGS (Krylov.jl default), CGS, CGS2 (classical Gram-Schmidt with reorthogonalisation).
#include "common.cuh"
#include <math.h>
#include <float.h>
#include <stdlib.h>
#include <algorithm>

namespace {
constexpr int GM_THREADS = 256;
constexpr int JT = 8;  // basis columns streamed together by the multi-dot kernel
constexpr int GM_KCAP = 16384;  // basis vectors per cycle: (GM_KCAP + 32) coefficients in shared memory, packed R = 1 GiB

struct GmresState {  // device-resident scalars
  int32_t status;    // 0 = running, else B200_LS_*
  int32_t k;         // Arnoldi iterations completed in the current cycle
  int32_t iter_base; // iterations completed in previous restart cycles
  int32_t itmax;
  int32_t kmax_cycle;  // restart length (or INT_MAX)
  int32_t pad;
  double rnorm0, rnorm, tol, atol, rtol, inv_h, hbis;
};

__device__ __forceinline__ void sym_givens(double a, double b, double& c, double& s, double& rho) {
  // Krylov.jl sym_givens (reflection form), restated in oracle/oracle.c the same way
  if (b == 0.0) {
    c = (a == 0.0) ? 1.0 : (a > 0 ? 1.0 : -1.0);
    s = 0.0;
    rho = fabs(a);
  } else if (a == 0.0) {
    c = 0.0;
    s = (b > 0 ? 1.0 : -1.0);
    rho = fabs(b);
  } else if (fabs(b) > fabs(a)) {
    const double t = a / b;
    s = (b > 0 ? 1.0 : -1.0) / sqrt(1.0 + t * t);
    c = s * t;
    rho = b / s;
  } else {
    const double t = b / a;
    c = (a > 0 ? 1.0 : -1.0) / sqrt(1.0 + t * t);
    s = c * t;
    rho = a / c;
  }
}

constexpr double GM_BREAKDOWN_TOL = 1.8189894035458565e-12;  // eps(Float64)^(3/4), Krylov.jl breakdown tolerance

// status after Arnoldi step k (1-based) of a cycle: 0 = go on, a B200_LS_* code, or -1 = cycle full (restart: the host resets)
__device__ __forceinline__ int gm_step_status(double rnorm, double hbis, int k, const GmresState* st) {
  if (!(rnorm == rnorm) || isinf(rnorm) || !(hbis == hbis) || isinf(hbis)) return B200_LS_NONFINITE;
  if (rnorm <= st->tol) return B200_LS_SOLVED;
  if (st->iter_base + k >= st->itmax) return B200_LS_MAXITERS;
  if (hbis <= GM_BREAKDOWN_TOL) return B200_LS_BREAKDOWN;
  if (k >= st->kmax_cycle) return -1;
  return 0;
}

__device__ __forceinline__ void block_rows(int64_t n, int64_t& r0, int64_t& r1) {
  // contiguous, even-aligned row range of this CTA
  int64_t chunk = (n + gridDim.x - 1) / gridDim.x;
  chunk = (chunk + 1) & ~(int64_t)1;
  r0 = (int64_t)blockIdx.x * chunk;
  r1 = r0 + chunk;
  if (r0 > n) r0 = n;
  if (r1 > n) r1 = n;
}

// ---- h[c] partials: partial[c * G + blockIdx.x] = sum over this CTA's rows of V[c][r] * w[r]
__global__ void __launch_bounds__(GM_THREADS) multidot_kernel(const GmresState* __restrict__ st, const double* const* __restrict__ V,
                                                               int k, const double* __restrict__ w, int64_t n,
                                                               double* __restrict__ partial) {
  if (st->status != 0) return;
  __shared__ double red[GM_THREADS / 32][JT];
  int64_t r0, r1;
  block_rows(n, r0, r1);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int G = gridDim.x;
  for (int c0 = 0; c0 < k; c0 += JT) {
    const double* vp[JT];
#pragma unroll
    for (int c = 0; c < JT; ++c) vp[c] = V[(c0 + c < k) ? (c0 + c) : c0];
    double acc[JT];
#pragma unroll
    for (int c = 0; c < JT; ++c) acc[c] = 0.0;
    for (int64_t r = r0 + 2 * threadIdx.x; r < r1; r += 2 * GM_THREADS) {
      if (r + 1 < r1) {
        const double2 w2 = *reinterpret_cast<const double2*>(w + r);
        double2 v2[JT];
#pragma unroll
        for (int c = 0; c < JT; ++c) {
          v2[c] = __ldcs(reinterpret_cast<const double2*>(vp[c] + r));  // streamed once: evict-first
        }
#pragma unroll
        for (int c = 0; c < JT; ++c) acc[c] = fma(v2[c].x, w2.x, fma(v2[c].y, w2.y, acc[c]));
      } else {
        const double w1 = w[r];
#pragma unroll
        for (int c = 0; c < JT; ++c) acc[c] = fma(vp[c][r], w1, acc[c]);
      }
    }
#pragma unroll
    for (int c = 0; c < JT; ++c) acc[c] = warp_sum(acc[c]);
    __syncthreads();
    if (lane == 0) {
#pragma unroll
      for (int c = 0; c < JT; ++c) red[wid][c] = acc[c];
    }
    __syncthreads();
    if (threadIdx.x < JT && c0 + threadIdx.x < k) {
      double s = 0.0;
#pragma unroll
      for (int q = 0; q < GM_THREADS / 32; ++q) s += red[q][threadIdx.x];
      partial[(int64_t)(c0 + threadIdx.x) * G + blockIdx.x] = s;
    }
  }
}

// ---- h[c] = sum_b partial[c*G + b] in fixed order (one warp per column).  accumulate: hacc[c] += h[c] (CGS2 second pass)
__global__ void __launch_bounds__(GM_THREADS) reduce_h_kernel(const GmresState* __restrict__ st, int k, int G,
                                                               const double* __restrict__ partial, double* __restrict__ h,
                                                               double* __restrict__ hacc) {
  if (st->status != 0) return;
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * (GM_THREADS / 32) + (threadIdx.x >> 5);
  if (c >= k) return;
  double s = 0.0;
  for (int b = lane; b < G; b += 32) s += partial[(int64_t)c * G + b];
  s = warp_sum(s);
  if (lane == 0) {
    h[c] = s;
    if (hacc) hacc[c] += s;
  }
}

// ---- w_out = w_in - sum_c coef[c] V[c]  (sign = -1)  or  w_in + sum_c coef[c] V[c] (sign = +1: x += V y);
//      optional ||w_out||^2 partial per CTA
__global__ void __launch_bounds__(GM_THREADS) update_kernel(const GmresState* __restrict__ st, int ignore_status,
                                                             const double* const* __restrict__ V, int k,
                                                             const double* __restrict__ coef, double sign,
                                                             const double* w_in, double* w_out, int64_t n,
                                                             double* __restrict__ norm_partial) {
  if (!ignore_status && st->status != 0) return;
  extern __shared__ double sh[];  // k coefficients + 32 reduction slots
  double* hc = sh;
  double* red = sh + k;
  for (int c = threadIdx.x; c < k; c += GM_THREADS) hc[c] = sign * coef[c];
  __syncthreads();
  int64_t r0, r1;
  block_rows(n, r0, r1);
  double nacc = 0.0;
  for (int64_t r = r0 + 2 * threadIdx.x; r < r1; r += 2 * GM_THREADS) {
    if (r + 1 < r1) {
      double2 w2 = *reinterpret_cast<const double2*>(w_in + r);
      int c = 0;
      for (; c + JT <= k; c += JT) {
        double2 v2[JT];
#pragma unroll
        for (int q = 0; q < JT; ++q) v2[q] = __ldcs(reinterpret_cast<const double2*>(V[c + q] + r));
#pragma unroll
        for (int q = 0; q < JT; ++q) {
          w2.x = fma(hc[c + q], v2[q].x, w2.x);
          w2.y = fma(hc[c + q], v2[q].y, w2.y);
        }
      }
      for (; c < k; ++c) {
        const double2 v2 = __ldcs(reinterpret_cast<const double2*>(V[c] + r));
        w2.x = fma(hc[c], v2.x, w2.x);
        w2.y = fma(hc[c], v2.y, w2.y);
      }
      *reinterpret_cast<double2*>(w_out + r) = w2;
      nacc = fma(w2.x, w2.x, fma(w2.y, w2.y, nacc));
    } else {
      double w1 = w_in[r];
      for (int c = 0; c < k; ++c) w1 = fma(hc[c], V[c][r], w1);
      w_out[r] = w1;
      nacc = fma(w1, w1, nacc);
    }
  }
  if (norm_partial) {
    nacc = block_sum(nacc, red);
    if (threadIdx.x == 0) norm_partial[blockIdx.x] = nacc;
  }
}

// ---- MGS fused pass i:  h_i = sum(partial_in) ; w -= h_i V[i] ; partial_out = (next ? V[next].w : ||w||^2)
//      i < 0: first pass, only the dot with V[0].
__global__ void __launch_bounds__(GM_THREADS) mgs_pass_kernel(const GmresState* __restrict__ st, const double* __restrict__ vi,
                                                               const double* __restrict__ vnext, int i,
                                                               const double* __restrict__ partial_in, double* __restrict__ partial_out,
                                                               double* __restrict__ h, double* __restrict__ w, int64_t n) {
  if (st->status != 0) return;
  __shared__ double red[32];
  __shared__ double hs;
  const int G = gridDim.x;
  double hi = 0.0;
  if (i >= 0) {
    double s = 0.0;
    for (int b = threadIdx.x; b < G; b += GM_THREADS) s += partial_in[b];
    s = block_sum(s, red);  // identical in every CTA: fixed summation tree
    if (threadIdx.x == 0) {
      hs = s;
      if (blockIdx.x == 0) h[i] = s;
    }
    __syncthreads();
    hi = hs;
  }
  int64_t r0, r1;
  block_rows(n, r0, r1);
  double acc = 0.0;
  for (int64_t r = r0 + 2 * threadIdx.x; r < r1; r += 2 * GM_THREADS) {
    if (r + 1 < r1) {
      double2 w2 = *reinterpret_cast<const double2*>(w + r);
      if (i >= 0) {
        const double2 v2 = __ldcs(reinterpret_cast<const double2*>(vi + r));
        w2.x = fma(-hi, v2.x, w2.x);
        w2.y = fma(-hi, v2.y, w2.y);
        *reinterpret_cast<double2*>(w + r) = w2;
      }
      if (vnext) {
        const double2 n2 = *reinterpret_cast<const double2*>(vnext + r);
        acc = fma(n2.x, w2.x, fma(n2.y, w2.y, acc));
      } else {
        acc = fma(w2.x, w2.x, fma(w2.y, w2.y, acc));
      }
    } else {
      double w1 = w[r];
      if (i >= 0) {
        w1 = fma(-hi, vi[r], w1);
        w[r] = w1;
      }
      acc = vnext ? fma(vnext[r], w1, acc) : fma(w1, w1, acc);
    }
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) partial_out[blockIdx.x] = acc;
}

// ---- start of a cycle: beta = sqrt(sum partial) ; tol (first cycle) ; z[0] = beta ; status
__global__ void __launch_bounds__(GM_THREADS) init_finish_kernel(GmresState* __restrict__ st, int G, const double* __restrict__ norm_partial,
                                                                  double* __restrict__ z, int first_cycle) {
  __shared__ double red[32];
  double s = 0.0;
  for (int b = threadIdx.x; b < G; b += GM_THREADS) s += norm_partial[b];
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const double beta = sqrt(s);
    if (first_cycle) {
      st->rnorm0 = beta;
      st->tol = st->atol + st->rtol * beta;
      st->iter_base = 0;
    }
    st->rnorm = beta;
    st->k = 0;
    z[0] = beta;
    st->inv_h = (beta > 0.0) ? 1.0 / beta : 0.0;
    if (!(beta == beta) || isinf(beta)) st->status = B200_LS_NONFINITE;
    else if (beta <= st->tol) st->status = B200_LS_SOLVED;
    else if (st->iter_base >= st->itmax) st->status = B200_LS_MAXITERS;
    else st->status = 0;
  }
}

// ---- end of Arnoldi step k (1-based): Hbis = sqrt(sum norm partials); apply the previous reflections to column k,
//      form the new one, update z / residual estimate / status.  R is packed upper triangular: column k at (k-1)k/2.
__global__ void __launch_bounds__(GM_THREADS) givens_kernel(GmresState* __restrict__ st, int k, int G, const double* __restrict__ norm_partial,
                                                             const double* __restrict__ h, double* __restrict__ R, double* __restrict__ cs,
                                                             double* __restrict__ sn, double* __restrict__ z, double* __restrict__ hraw) {
  if (st->status != 0) return;
  __shared__ double red[32];
  double s = 0.0;
  for (int b = threadIdx.x; b < G; b += GM_THREADS) s += norm_partial[b];
  s = block_sum(s, red);
  double* Rk = R + (int64_t)(k - 1) * k / 2;
  for (int i = threadIdx.x; i < k; i += GM_THREADS) Rk[i] = h[i];
  if (hraw) {  // raw Hessenberg column for parity tests: k+1 entries at offset (k-1)(k+2)/2
    double* hr = hraw + (int64_t)(k - 1) * (k + 2) / 2;
    for (int i = threadIdx.x; i < k; i += GM_THREADS) hr[i] = h[i];
    if (threadIdx.x == 0) hr[k] = sqrt(s);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const double hbis = sqrt(s);
    for (int i = 0; i + 1 < k; ++i) {
      const double rt = cs[i] * Rk[i] + sn[i] * Rk[i + 1];
      Rk[i + 1] = sn[i] * Rk[i] - cs[i] * Rk[i + 1];
      Rk[i] = rt;
    }
    double c, s_, rho;
    sym_givens(Rk[k - 1], hbis, c, s_, rho);
    cs[k - 1] = c;
    sn[k - 1] = s_;
    Rk[k - 1] = rho;
    const double zeta = s_ * z[k - 1];
    z[k - 1] = c * z[k - 1];
    z[k] = zeta;
    const double rnorm = fabs(zeta);
    st->rnorm = rnorm;
    st->hbis = hbis;
    st->k = k;
    st->inv_h = (hbis > 0.0) ? 1.0 / hbis : 0.0;
    st->status = gm_step_status(rnorm, hbis, k, st);
  }
}

// ---- V[k] = w * inv_h
__global__ void __launch_bounds__(GM_THREADS) normalize_kernel(const GmresState* __restrict__ st, int require_running,
                                                                const double* __restrict__ w, double* __restrict__ v, int64_t n) {
  if (require_running && st->status != 0) return;
  const double s = st->inv_h;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x * 2;
  for (int64_t r = 2 * ((int64_t)blockIdx.x * blockDim.x + threadIdx.x); r < n; r += stride) {
    if (r + 1 < n) {
      double2 w2 = *reinterpret_cast<const double2*>(w + r);
      w2.x *= s;
      w2.y *= s;
      *reinterpret_cast<double2*>(v + r) = w2;
    } else {
      v[r] = w[r] * s;
    }
  }
}

// ---- y = R^{-1} z for the first k columns (single CTA, column-oriented back substitution)
__global__ void __launch_bounds__(GM_THREADS) backsolve_kernel(const GmresState* __restrict__ st, const double* __restrict__ R,
                                                                const double* __restrict__ z, double* __restrict__ y, int kcap) {
  const int k = st->k;
  extern __shared__ double zs[];
  for (int i = threadIdx.x; i < k; i += GM_THREADS) zs[i] = z[i];
  __syncthreads();
  for (int i = k - 1; i >= 0; --i) {
    const double* Ri = R + (int64_t)i * (i + 1) / 2;
    const double d = Ri[i];
    const double yi = (d == 0.0) ? 0.0 : zs[i] / d;
    __syncthreads();
    if (threadIdx.x == 0) zs[i] = yi;
    for (int j = threadIdx.x; j < i; j += GM_THREADS) zs[j] -= Ri[j] * yi;
    __syncthreads();
  }
  for (int i = threadIdx.x; i < kcap; i += GM_THREADS) y[i] = (i < k) ? zs[i] : 0.0;
}

__global__ void __launch_bounds__(GM_THREADS) residual_init_kernel(int64_t n, const double* __restrict__ b, const double* __restrict__ Ax,
                                                                    double* __restrict__ r, double* __restrict__ norm_partial) {
  __shared__ double red[32];
  double acc = 0.0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const double v = Ax ? b[i] - Ax[i] : b[i];
    r[i] = v;
    acc = fma(v, v, acc);
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) norm_partial[blockIdx.x] = acc;
}

// ---- generic operator kernels (b2/b3 plug-in points): CSC matrix through a row view (deterministic gather: the scatter form
//      with atomicAdd it replaces summed in a run-dependent order) and dense column-major GEMV
__global__ void __launch_bounds__(GM_THREADS) csc_rows_spmv_kernel(int64_t n, const int64_t* __restrict__ rowptr, const int64_t* __restrict__ col,
                                                                    const int64_t* __restrict__ map, const double* __restrict__ nzval,
                                                                    const double* __restrict__ x, double* __restrict__ y) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  double s = 0.0;
  for (int64_t e = rowptr[r]; e < rowptr[r + 1]; ++e) s = fma(nzval[map[e]], x[col[e]], s);  // ascending column order
  y[r] = s;
}
__global__ void __launch_bounds__(GM_THREADS) dense_gemv_kernel(int trans, int64_t m, int64_t n, const double* __restrict__ A, int64_t ld,
                                                                 const double* __restrict__ x, double* __restrict__ y) {
  __shared__ double red[32];
  if (!trans) {  // y = A x: thread per row, coalesced down the column
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    double s = 0.0;
    for (int64_t c = 0; c < n; ++c) s = fma(A[c * ld + i], x[c], s);
    y[i] = s;
  } else {  // y = A' x: CTA per column
    for (int64_t c = blockIdx.x; c < n; c += gridDim.x) {
      double s = 0.0;
      for (int64_t i = threadIdx.x; i < m; i += blockDim.x) s = fma(A[c * ld + i], x[i], s);
      s = block_sum(s, red);
      if (threadIdx.x == 0) y[c] = s;
      __syncthreads();
    }
  }
}
// y = A' x for a TALL, SKINNY A (m rows >> n <= TG_NC columns: the n x threshold factors of LimitedMemoryBroyden): every CTA takes a
// row range and all columns in one pass (x read once), partials summed in a fixed order by a second kernel — deterministic, no atomics
constexpr int TG_NC = 16;
__global__ void __launch_bounds__(GM_THREADS) tall_gemvt_partial_kernel(int64_t m, int nc, const double* __restrict__ A, int64_t ld, const double* __restrict__ x,
                                                                         double* __restrict__ partial) {
  __shared__ double red[GM_THREADS / 32][TG_NC];
  const int G = gridDim.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t per = (m + G - 1) / G, r0 = (int64_t)blockIdx.x * per, r1 = min(m, r0 + per);
  double acc[TG_NC];
#pragma unroll
  for (int c = 0; c < TG_NC; ++c) acc[c] = 0.0;
  for (int64_t r = r0 + threadIdx.x; r < r1; r += GM_THREADS) {
    const double xr = x[r];
#pragma unroll
    for (int c = 0; c < TG_NC; ++c)
      if (c < nc) acc[c] = fma(A[(int64_t)c * ld + r], xr, acc[c]);
  }
#pragma unroll
  for (int c = 0; c < TG_NC; ++c) acc[c] = warp_sum(acc[c]);
  if (lane == 0) {
#pragma unroll
    for (int c = 0; c < TG_NC; ++c) red[wid][c] = acc[c];
  }
  __syncthreads();
  if (threadIdx.x < nc) {
    double s = 0.0;
    for (int q = 0; q < GM_THREADS / 32; ++q) s += red[q][threadIdx.x];
    partial[(int64_t)threadIdx.x * G + blockIdx.x] = s;
  }
}
__global__ void tall_gemvt_final_kernel(int nc, int G, const double* __restrict__ partial, double* __restrict__ y) {
  const int c = threadIdx.x;
  if (c >= nc) return;
  double s = 0.0;
  for (int g = 0; g < G; ++g) s += partial[(int64_t)c * G + g];
  y[c] = s;
}
// =====================================================================================================================
// Resident Arnoldi step (engine B200_ENGINE_RESIDENT): ONE cooperative kernel per Arnoldi iteration for the built-in
// Brusselator operators (or an assembled sparse Jacobian through its CSR view).  One CTA per SM; CTA b owns the cells
// [b*cpc, (b+1)*cpc) of both species for the whole step:
//   1. w = J(u) v_k is evaluated straight into registers — it never touches HBM;
//   2. the Krylov basis is streamed ONCE per Gram-Schmidt pass (TMA bulk copies into two shared-memory stages + a third
//      stage in registers); per basis vector: dot partial -> cross-CTA exchange -> w -= h_i v_i from the copy still on
//      chip.  That is modified Gram-Schmidt (Krylov.jl's scheme), applied twice when reorthogonalisation is requested:
//      `passes * k * Bv` of HBM traffic instead of the 2x of the multi-kernel engine;
//   3. ||w||, Givens recurrence (CTA 0), normalisation and the store of v_{k+1} close the step.
// Cross-CTA exchanges poll with bounded spins so a fault can never hang the GPU (cooperative launch guarantees co-residency).
struct ResidentParams {
  int dim, N, k, passes, G;
  int opkind;       // 0: built-in Brusselator J(u) v, 1: assembled sparse matrix through its CSR view
  const int64_t *rowptr, *csr_col, *csr_map;
  const double* nzval;
  int64_t NC;       // cells (opkind 1: half of the rows — the row set is split in two contiguous segments the same way)
  int cpc;          // cells per CTA (even)
  int qs;           // row pairs per thread held by each shared-memory stage (the rest is read from global memory)
  double a, A;
  const double* u;
  const double* const* V;
  double* vnew;     // V[k]
  unsigned long long* slots;  // four rotating exchange tables of {data32 | epoch << 32} words (NCCL-LL style flag-in-word publication)
  unsigned epoch_base;        // unique, monotonically increasing across launches
  int* err;
  double* h;        // Hessenberg column workspace (k + 1)
  double* gsub;     // r3g kernel: gsub[i] = <v_i, v_{i-1}>, written by the step that creates v_i
  double *R, *cs, *sn, *z, *hraw;
  GmresState* st;
};

// Cross-CTA exchange: flag-in-word tables (common.cuh), one entry per CTA, published with ll_store.  The polls below keep their
// own loops: rewritten on ll_load / ll_wait they changed the kernel's code and measured slower.
constexpr int LL_MAXG = 160;                     // CTAs an exchange table has room for
constexpr int R3_POLLERS = LL_MAXG;              // threads 0 .. R3_POLLERS-1 poll one table entry each (5 warps)
constexpr int R3_SPARE_POLLER = R3_POLLERS - 1;  // fetches the Gram sub-diagonal entry instead: at most R3_SPARE_POLLER CTAs
constexpr int R3_THREADS = 256;
// CTA 0: Hessenberg column -> packed R with the stored Givens rotations, new rotation, residual norm, status (same recurrence
// as givens_kernel).  The recurrence is serial in i, so one thread runs it — but on a shared-memory copy of the column and of the
// stored rotations that the whole CTA stages first (and writes back afterwards): run straight on global memory every iteration
// waits for an L2 round trip (the stores to R may alias the rotations, so the loads cannot be hoisted), a fixed cost x k per step.
// `ws` = the stage buffers, free once the sweep is over (cap doubles).
__device__ __forceinline__ void resident_givens_tail(const ResidentParams& P, double hbis, double inv, double* ws, int cap, int tid) {
  const int k = P.k;
  GmresState* st = P.st;
  double* Rk = P.R + (int64_t)(k - 1) * k / 2;
  double* hr = P.hraw ? P.hraw + (int64_t)(k - 1) * (k + 2) / 2 : nullptr;
  const bool staged = 3 * k <= cap;
  double *col, *cs, *sn;
  if (staged) {
    col = ws; cs = ws + k; sn = ws + 2 * k;
    for (int i = tid; i < k; i += R3_THREADS) {
      const double h = P.h[i];
      col[i] = h; cs[i] = P.cs[i]; sn[i] = P.sn[i];
      if (hr) hr[i] = h;
    }
    __syncthreads();
  } else {
    col = Rk; cs = P.cs; sn = P.sn;
    if (tid == 0) {
      for (int i = 0; i < k; ++i) { const double h = P.h[i]; Rk[i] = h; if (hr) hr[i] = h; }
    }
  }
  if (tid == 0) {
    if (hr) hr[k] = hbis;
    double x = col[0];
    for (int i = 0; i + 1 < k; ++i) {
      const double nx = col[i + 1];
      col[i] = cs[i] * x + sn[i] * nx;
      x = sn[i] * x - cs[i] * nx;
    }
    double c, s_, rho;
    sym_givens(x, hbis, c, s_, rho);
    P.cs[k - 1] = c; P.sn[k - 1] = s_; col[k - 1] = rho;
    const double zeta = s_ * P.z[k - 1];
    P.z[k - 1] = c * P.z[k - 1];
    P.z[k] = zeta;
    const double rnorm = fabs(zeta);
    st->rnorm = rnorm; st->hbis = hbis; st->k = k; st->inv_h = inv;
    st->status = *P.err ? B200_LS_NONFINITE : gm_step_status(rnorm, hbis, k, st);  // an exchange timed out: report, stop
  }
  if (staged) {
    __syncthreads();
    for (int i = tid; i < k; i += R3_THREADS) Rk[i] = col[i];
  }
}

// =====================================================================================================================
// Three-stage, lag-1 organisation of the resident Arnoldi step (rows of one SM fit 60 per thread at 256 threads): the two
// shared-memory stages are joined by a THIRD stage held in registers (32 more doubles per thread, filled by 128-bit global
// loads that stay in flight for a whole step, + a cp.async annex), so three basis vectors are on chip and the
// exchange of vector t overlaps the dot products of vector t+1:
//     h_{t+1} = <v_{t+1}, w_t> - h_t <v_{t+1}, v_t>          (w_t: w before the update with v_t)
// which are the modified Gram-Schmidt coefficients exactly (the cross product restores the missing update); the pair
// (<v_{t+1}, w_t>, <v_{t+1}, v_t>) is published before h_t is known.  Stage roles rotate with t mod 3 (0, 1: shared memory
// via TMA bulk copies, 2: registers).  Exchange: replicated pull tables (16 replicas, 32-byte entries {a, c} with the epoch
// in every 64-bit word), one entry per polling thread; four table buffers rotate.
// Capacity: at N = 100 on the 132 SMs of an H100 a CTA owns 15 152 rows, and w plus three whole vectors (485 KB) exceed what
// one SM holds (64K registers + 227 KB of shared memory).  The shared-memory stages therefore keep the first `qs` row pairs of
// every thread (the prefix of the CTA's rows that fits beside the annex); the pairs q >= qs of those two stages (the global
// tail, 9 per thread at N = 100) are needed at each of their two uses, the dot sweep of step t-1 and the update sweep of step t.
// With the register file full, a tail pair read straight from global memory is one dependent L2 round trip; instead the tail
// is copied by 16-byte cp.async, all pairs in flight together, into stage slots the thread has released (R3_SLOTGET):
//   update sweep of v_t (shared-memory role): once pairs 0 .. R3_TAIL_AT-1 are applied, their slots of v_t's own stage are
//     free; the tail lands there while pairs R3_TAIL_AT .. qs-1 are applied, and is applied last (the pair order is unchanged);
//   dot sweep of v_{t+1} when it is stage 0's (t = 2 mod 3): the tail lands in stage 1, released by v_{t-1} one step before,
//     whose refill with v_{t+2} waits until every thread has passed the barrier after that dot sweep (an L2 prefetch of the
//     whole of v_{t+2} keeps the old place).  The dot sweep of stage 1's vectors has no released slots (stage 0 holds v_t,
//     the annex v_{t+2}) and reads its tail from global memory.
// Which tail pairs have a slot: r3_update_slot / r3_dot_slot below; the others are read directly.
// cp.async groups of a thread, in commit order over one rotation (steps t = 0, 1, 2 mod 3):
//   end of a role-2 step:  R, the register stage's annex of v_{t+3};
//   role-0 step:           U0, the update-sweep tail of v_t; its wait (inside the sweep) also completes R, issued half a
//                          step earlier;
//   role-1 step:           the wait at its start (register stage of v_{t+1}) finds R complete; U1 is committed and waited
//                          inside the update sweep; D, the dot-sweep tail of v_{t+2}, is committed at its end;
//   role-2 step:           D alone is pending at the wait inside the dot sweep.
// At most two groups are ever pending; the only wait that completes a group other than its sweep's own is U0's (R).
constexpr int R3_RP = 30;            // row pairs per thread
constexpr int R3_ROWS = 2 * R3_RP;   // 60 rows per thread -> at most 15360 rows (7680 cells) per CTA
constexpr int R3_RPR = 16;           // pairs of the third stage held in registers; the last R3_RP - R3_RPR pairs of each thread
constexpr int R3_VR = 2 * R3_RPR;    //   sit in a shared-memory annex filled by cp.async (register budget: 255, no spills)
constexpr size_t R3_ANNEX_BYTES = (size_t)(R3_RP - R3_RPR) * R3_THREADS * 16;
constexpr int R3_REPL = 16;
constexpr size_t R3_BUF_WORDS = (size_t)R3_REPL * LL_MAXG * 4;

constexpr unsigned R3_SPIN_BOUND = 1u << 22;  // exchange polls give up (and flag P.err) after this many reloads

// warp 0: CTA b's entry {a, c} of exchange table `buf`, in every replica
__device__ __forceinline__ void r3_post(unsigned long long* buf, int b, double a, double c, unsigned epoch) {
  const int lane = threadIdx.x;
  if (lane < R3_REPL) {
    unsigned long long* dst = buf + ((size_t)lane * LL_MAXG + b) * 4;
    ll_store(dst, (unsigned long long)__double_as_longlong(a), epoch);
    ll_store(dst + 2, (unsigned long long)__double_as_longlong(c), epoch);
  }
}
// threads 0 .. R3_POLLERS-1 poll one entry each, both pairs in flight together; per-warp partial sums land in gA / gC (5 each); caller synchronises
__device__ __forceinline__ void r3_poll(const unsigned long long* buf, int b, int G, unsigned epoch, int* err, double* gA, double* gC) {
  const int tid = threadIdx.x;
  if (tid < R3_POLLERS) {
    double xa = 0.0, xc = 0.0;
    if (tid < G) {
      const unsigned long long* src = buf + ((size_t)(b & (R3_REPL - 1)) * LL_MAXG + tid) * 4;
      unsigned long long a0, a1, c0, c1;
      unsigned spins = 0;
      bool ok;
      do {
        asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(a0), "=l"(a1) : "l"(src) : "memory");
        asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(c0), "=l"(c1) : "l"(src + 2) : "memory");
        ok = ((unsigned)(a0 >> 32) == epoch) && ((unsigned)(a1 >> 32) == epoch) && ((unsigned)(c0 >> 32) == epoch) && ((unsigned)(c1 >> 32) == epoch);
        if (++spins > R3_SPIN_BOUND) { *err = 1; break; }
      } while (!ok);
      xa = __longlong_as_double((long long)((a0 & 0xffffffffull) | (a1 << 32)));
      xc = __longlong_as_double((long long)((c0 & 0xffffffffull) | (c1 << 32)));
    }
    xa = warp_sum(xa);
    xc = warp_sum(xc);
    if ((tid & 31) == 0) { gA[tid >> 5] = xa; gC[tid >> 5] = xc; }
  }
}

struct R3Ctx {
  double *stage0, *stage1;
  double2* annex;
  int nrow, ncell, total, k, b, G;
  int qs;  // row pairs per thread held by the shared-memory stages (>= 1)
};

// The shared-memory stages hold the CTA's rows [0, 2 * R3_THREADS * qs): a prefix of the first species' segment, or all of it
// and a prefix of the second species' segment.  The rows past the stage (the global tail) are prefetched into L2 here, so that
// their copies into stage slots and the direct reads of the stage-1 dot sweep end in L2 instead of HBM.  The copy reads
// evict-first: the rows it copies are not needed again in this launch.
__device__ __forceinline__ void r3_issue_smem(const ResidentParams& P, const R3Ctx& cx, uint64_t* mbar, int t, int stage) {
  if (threadIdx.x == 0 && cx.nrow > 0) {
    const double* src = P.V[t % cx.k];
    double* dst = stage ? cx.stage1 : cx.stage0;
    const int srow = min(cx.nrow, 2 * R3_THREADS * cx.qs);
    const int r0 = min(srow, cx.ncell), r1 = srow - r0;
    const int64_t c0 = (int64_t)cx.b * P.cpc;
    const uint64_t pol = l2_evict_first_policy();
    mbar_expect_tx(&mbar[stage], (unsigned)srow * 8u);
    tma_bulk_load(dst, src + c0, (unsigned)r0 * 8u, &mbar[stage], pol);
    if (r1 > 0) tma_bulk_load(dst + cx.ncell, src + P.NC + c0, (unsigned)r1 * 8u, &mbar[stage], pol);
    // rows [srow, nrow): the rest of the first species' segment, then the second species' rows from max(srow, ncell) on
    // (even bounds: every range is a multiple of 16 bytes)
    if (srow < cx.ncell) l2_bulk_prefetch(src + c0 + srow, (unsigned)(cx.ncell - srow) * 8u);
    if (srow < cx.nrow) {
      const int a = max(srow, cx.ncell) - cx.ncell;
      l2_bulk_prefetch(src + P.NC + c0 + a, (unsigned)(cx.ncell - a) * 8u);
    }
  }
}
// element pair q (offset lr from this thread's first pair) of a shared-memory-role vector: from the stage `sp` when it holds
// the pair, else from the vector itself in global memory (`gp` = its first element of this thread, lims / hop as in r3_issue_regs)
#define R3_SMGET(q, lr, sp, gp, o0, o1)                                                                                         \
  do {                                                                                                                            \
    double2 z_;                                                                                                                   \
    if ((q) < cx.qs) z_ = *reinterpret_cast<const double2*>((sp) + (lr));                                                         \
    else z_ = __ldg(reinterpret_cast<const double2*>((gp) + (lr) + (((lr) >= lims) ? hop : (int64_t)0)));                        \
    o0 = z_.x; o1 = z_.y;                                                                                                         \
  } while (0)
// the same when tail pair q, if `slot`, was copied by r3_tail_copy into slot q - qs of stage `tp` (this thread's first
// element); the thread's cp.async groups are waited for at the first of them, q = qs
#define R3_SLOTGET(q, lr, sp, tp, slot, gp, o0, o1)                                                                             \
  do {                                                                                                                            \
    double2 z_;                                                                                                                   \
    if ((q) < cx.qs) z_ = *reinterpret_cast<const double2*>((sp) + (lr));                                                         \
    else if (slot) {                                                                                                              \
      if ((q) == cx.qs) asm volatile("cp.async.wait_group 0;" ::: "memory");                                                     \
      z_ = *reinterpret_cast<const double2*>((tp) + (lr) - 2 * R3_THREADS * cx.qs);                                               \
    } else z_ = __ldg(reinterpret_cast<const double2*>((gp) + (lr) + (((lr) >= lims) ? hop : (int64_t)0)));                     \
    o0 = z_.x; o1 = z_.y;                                                                                                         \
  } while (0)
// L2 prefetch of all of this CTA's rows of vector t (both species' segments)
__device__ __forceinline__ void r3_prefetch_l2(const ResidentParams& P, const R3Ctx& cx, int t) {
  if (threadIdx.x == 0 && cx.nrow > 0) {
    const double* src = P.V[t % cx.k] + (int64_t)cx.b * P.cpc;
    l2_bulk_prefetch(src, (unsigned)cx.ncell * 8u);
    l2_bulk_prefetch(src + P.NC, (unsigned)cx.ncell * 8u);
  }
}
// Slots of the global tail (pairs q >= qs at slot q - qs, nslot <= qs of them): every released slot in the dot sweep of a
// stage-0 vector; in an update sweep, the slots of pairs 0 .. R3_TAIL_AT-1, and only when the copy is issued before the first
// tail pair is needed (qs >= R3_TAIL_AT).  The update sweep issues its copy at one compile-time place, after pair R3_TAIL_AT-1:
// a place that depends on qs at run time costs registers the kernel does not have (it spills).  R3_TAIL_AT = 9 covers the
// whole tail of the stock split at N = 100 (qs = 21 of 30 pairs) and of every split from qs = 21 on.
constexpr int R3_TAIL_AT = 9;
// whether tail pair q (>= qs, compile-time after unrolling) sits in a slot, written as comparisons of qs with constants
// (a slot bound held in a register costs one the kernel does not have)
__device__ __forceinline__ bool r3_dot_slot(const R3Ctx& cx, int q) { return cx.qs > q / 2; }  // q < 2 qs
__device__ __forceinline__ bool r3_update_slot(const R3Ctx& cx, int q) { return cx.qs >= R3_TAIL_AT && cx.qs > q - R3_TAIL_AT; }
// this thread's global-tail pairs q = qs .. qs + nslot - 1 of a vector (`gp` = its first element of this thread, lim / lims /
// hop as in r3_issue_regs) -> slots 0 .. nslot-1 of a stage (`ts` = the stage + 2 * tid), one cp.async group.  Every source
// lies in this CTA's rows of one species' segment; sources and slots are 16-byte aligned (even offsets of aligned bases).
// Call only when the thread has a tail pair (lim > 2 * R3_THREADS * qs): the group it commits is waited on in R3_SLOTGET.
// LAST: the copy of the update sweep, the tail's last use in this launch, reads evict-first; the copy for the dot sweep
// (LAST = false) reads with the default policy, so that the tail is still in L2 for the update sweep one step later.
template <bool LAST = true>
__device__ __forceinline__ void r3_tail_copy(const R3Ctx& cx, const double* gp, double* ts, int nslot, int lim, int lims, int64_t hop) {
  const uint64_t pol = LAST ? l2_evict_first_policy() : 0;
  for (int j = 0; j < nslot; ++j) {
    const int lr = 2 * R3_THREADS * (cx.qs + j);
    if (lr >= lim) break;  // also ends the copy at pair R3_RP - 1
    const double* src = gp + lr + ((lr >= lims) ? hop : (int64_t)0);
    if (LAST) cp_async16(ts + 2 * R3_THREADS * j, src, pol);
    else cp_async16(ts + 2 * R3_THREADS * j, src);
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
}
__device__ __forceinline__ void r3_issue_regs(const ResidentParams& P, const R3Ctx& cx, int t, double (&vr)[R3_VR]) {
  // thread-relative form (constant offsets, two per-thread limits) so that nothing per-q stays live across the step
  const double* src = P.V[t % cx.k] + (int64_t)cx.b * P.cpc + 2 * (int)threadIdx.x;
  const int lim = cx.nrow - 2 * (int)threadIdx.x, lims = cx.ncell - 2 * (int)threadIdx.x;
  const int64_t hop = P.NC - cx.ncell;  // from the end of this CTA's first-species segment to the start of its second
  const uint64_t pol = l2_evict_first_policy();  // the vector is read once in this launch
#pragma unroll
  for (int q = 0; q < R3_RP; ++q) {
    const int lr = 2 * R3_THREADS * q;
    const double* p = src + ((lr >= lims) ? hop : (int64_t)0) + lr;
    if (q < R3_RPR) {
      if (lr < lim)
        asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.f64 {%0, %1}, [%2], %3;"
                     : "=d"(vr[2 * (q < R3_RPR ? q : 0)]), "=d"(vr[2 * (q < R3_RPR ? q : 0) + 1]) : "l"(p), "l"(pol));
    } else if (lr < lim) {
      cp_async16(cx.annex + (q - R3_RPR) * R3_THREADS + threadIdx.x, p, pol);
    }
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
}
// element pair q of the third stage (compile-time q after unrolling)
#define R3_VRGET(q, o0, o1)                                                                            \
  do {                                                                                                 \
    if ((q) < R3_RPR) { o0 = vr[2 * ((q) < R3_RPR ? (q) : 0)]; o1 = vr[2 * ((q) < R3_RPR ? (q) : 0) + 1]; } \
    else { const double2 z_ = cx.annex[((q) - R3_RPR) * R3_THREADS + threadIdx.x]; o0 = z_.x; o1 = z_.y; }     \
  } while (0)

// w = J(u) v_k (built-in Brusselator tangent) or the assembled sparse matrix times v_k (CSR view) for this CTA's rows;
// thread `tid` holds the row pairs 2 * (tid + R3_THREADS * q), q = 0 .. R3_RP-1, of the CTA's row slice
__device__ __forceinline__ void r3_apply_operator(const ResidentParams& P, const R3Ctx& cx, double (&w)[R3_ROWS]) {
  const int tid = threadIdx.x;
  const double* vk = P.V[P.k - 1];
  const int N = P.N;
  const int64_t NC = P.NC;
  const int ncell = cx.ncell, nrow = cx.nrow;
  const int64_t c0 = (int64_t)cx.b * P.cpc;
  if (P.opkind == 1) {  // assembled sparse matrix through its CSR view: a gather per row
#pragma unroll
    for (int qq = 0; qq < R3_ROWS; ++qq) {
      const int lr = 2 * (tid + R3_THREADS * (qq >> 1)) + (qq & 1);
      w[qq] = 0.0;
      if (lr < nrow) {
        const int s = lr >= ncell;
        const int64_t r = (int64_t)s * NC + c0 + (lr - s * ncell);
        double acc = 0.0;
        for (int64_t e = P.rowptr[r], e1 = P.rowptr[r + 1]; e < e1; ++e) acc = fma(P.nzval[P.csr_map[e]], vk[P.csr_col[e]], acc);
        w[qq] = acc;
      }
    }
    return;
  }
  // Built-in Brusselator J(u) v, a PAIR of neighbouring cells per step (the pair never straddles a grid row: the cell count per
  // CTA and N are even), 16-byte loads for everything but the two i-neighbours outside the pair.  Cell coordinates come from two
  // multiplications by reciprocals, exact for these ranges ((c + 1/2) / d is never within 2^-21 of an integer, the product's error
  // is < 2^-40) instead of an int64 and an int32 division per row, a fixed cost of every Arnoldi step whatever the basis size.
  const int N2 = N * N, c0i = (int)c0;
  const double invN = 1.0 / (double)N, invN2 = 1.0 / (double)N2;
  const bool d3 = P.dim == 3;
  const double* __restrict__ uu_ = P.u;
#pragma unroll
  for (int q = 0; q < R3_RP; ++q) {
    const int lr = 2 * (tid + R3_THREADS * q);
    w[2 * q] = 0.0;
    w[2 * q + 1] = 0.0;
    if (lr < nrow) {
      const int s = lr >= ncell;
      const int c = c0i + (lr - s * ncell);  // even
      int i, j, kk = 0;
      if (d3) {
        kk = (int)(((double)c + 0.5) * invN2);
        const int r = c - kk * N2;
        j = (int)(((double)r + 0.5) * invN);
        i = r - j * N;
      } else {
        j = (int)(((double)c + 0.5) * invN);
        i = c - j * N;
      }
      const double* x = vk + (int64_t)s * NC + c;
      const double2 xc = *reinterpret_cast<const double2*>(x);
      const double xl = x[(i == 0) ? (N - 1) : -1];
      const double xr = x[(i + 2 == N) ? (2 - N) : 2];
      const int ojm = (j == 0) ? (N - 1) * N : -N, ojp = (j + 1 == N) ? -(N - 1) * N : N;
      const double2 xjm = *reinterpret_cast<const double2*>(x + ojm), xjp = *reinterpret_cast<const double2*>(x + ojp);
      double lap0 = xl + xc.y + xjp.x + xjm.x - 4.0 * xc.x;
      double lap1 = xc.x + xr + xjp.y + xjm.y - 4.0 * xc.y;
      if (d3) {
        const int okm = (kk == 0) ? (N - 1) * N2 : -N2, okp = (kk + 1 == N) ? -(N - 1) * N2 : N2;
        const double2 xkm = *reinterpret_cast<const double2*>(x + okm), xkp = *reinterpret_cast<const double2*>(x + okp);
        lap0 = lap0 + (xkp.x + xkm.x - 2.0 * xc.x);
        lap1 = lap1 + (xkp.y + xkm.y - 2.0 * xc.y);
      }
      const double2 u2 = *reinterpret_cast<const double2*>(uu_ + c), v2 = *reinterpret_cast<const double2*>(uu_ + NC + c);
      const double2 d2 = *reinterpret_cast<const double2*>(vk + c), e2 = *reinterpret_cast<const double2*>(vk + NC + c);
      const double uv0 = 2.0 * u2.x * v2.x, uu0 = u2.x * u2.x, uv1 = 2.0 * u2.y * v2.y, uu1 = u2.y * u2.y;
      w[2 * q] = s ? (P.a * lap0 + (P.A - uv0) * d2.x - uu0 * e2.x) : (P.a * lap0 + (uv0 - (P.A + 1.0)) * d2.x + uu0 * e2.x);
      w[2 * q + 1] = s ? (P.a * lap1 + (P.A - uv1) * d2.y - uu1 * e2.y) : (P.a * lap1 + (uv1 - (P.A + 1.0)) * d2.y + uu1 * e2.y);
    }
  }
}

// Early poll of exchange t: the words were published one step ago, so the load is issued BEFORE the dot sweep of the
// step and its L2 round trip is hidden underneath it; r3g_poll_finish checks the epochs afterwards and only spins if a CTA is late.
__device__ __forceinline__ void r3g_poll_issue(const unsigned long long* buf, int b, int G, unsigned long long& a0, unsigned long long& a1) {
  const int tid = threadIdx.x;
  a0 = 0ull; a1 = 0ull;
  if (tid < G) {
    const unsigned long long* src = buf + ((size_t)(b & (R3_REPL - 1)) * LL_MAXG + tid) * 4;
    asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(a0), "=l"(a1) : "l"(src) : "memory");
  }
}
__device__ __forceinline__ void r3g_poll_finish(const unsigned long long* buf, int b, int G, unsigned epoch, int* err, bool need_c, unsigned long long a0,
                                                unsigned long long a1, double* gA, double* gC) {
  const int tid = threadIdx.x;
  if (tid < R3_POLLERS) {
    double xa = 0.0, xc = 0.0;
    if (tid < G) {
      const unsigned long long* src = buf + ((size_t)(b & (R3_REPL - 1)) * LL_MAXG + tid) * 4;
      unsigned spins = 0;
      while (((unsigned)(a0 >> 32) != epoch) || ((unsigned)(a1 >> 32) != epoch)) {
        asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(a0), "=l"(a1) : "l"(src) : "memory");
        if (++spins > R3_SPIN_BOUND) { *err = 1; break; }
      }
      xa = __longlong_as_double((long long)((a0 & 0xffffffffull) | (a1 << 32)));
      if (need_c) {  // wrap-around step only: the cross product travels in the second pair (same store burst as the first)
        unsigned long long c0, c1;
        spins = 0;
        do {
          asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(c0), "=l"(c1) : "l"(src + 2) : "memory");
          if (++spins > R3_SPIN_BOUND) { *err = 1; break; }
        } while (((unsigned)(c0 >> 32) != epoch) || ((unsigned)(c1 >> 32) != epoch));
        xc = __longlong_as_double((long long)((c0 & 0xffffffffull) | (c1 << 32)));
      }
    }
    xa = warp_sum(xa);
    if ((tid & 31) == 0) gA[tid >> 5] = xa;
    if (need_c) {
      xc = warp_sum(xc);
      if ((tid & 31) == 0) gC[tid >> 5] = xc;
    }
  }
}

struct R3GShared {
  uint64_t mbar[2];
  double redA[2][8], redC[2][8];  // per-warp partials of the dot sweep, by step parity
  double gA[2][8], gC[2][8];      // per-warp sums of the polled exchange entries, by step parity; gC[.][5] = stored cross product
  double hprev[2];                // previous Gram-Schmidt coefficient, by step parity (kept out of the register file)
};
static_assert(R3_THREADS == 8 * 32 && R3_POLLERS == 5 * 32, "sum8 / sum5 add the per-warp partials of the CTA / of the polling warps");
// the fixed summation orders of the per-warp partials (every CTA adds the same numbers in the same order)
__device__ __forceinline__ double sum8(const double* r) { return ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7])); }
__device__ __forceinline__ double sum5(const double* g) { return ((g[0] + g[1]) + (g[2] + g[3])) + g[4]; }

// TAIL: this CTA has a global tail (rows past its stages).  Without one (N <= 88 on an H100) the step compiles to the plain
// three-stage rotation, with none of the tail's branches in its sweeps.
template <int ROLE, bool TAIL>
__device__ __forceinline__ void r3g_step(const ResidentParams& P, R3Ctx& cx, R3GShared& sh, int t, double (&w)[R3_ROWS], double (&vr)[R3_VR]) {
  constexpr int NEXT = (ROLE + 1) % 3;
  const int tid = threadIdx.x;
  const int par = t & 1;
  const int lim = cx.nrow - 2 * tid;                       // row pair q of this thread exists iff 2 * R3_THREADS * q < lim
  double* const sc = (ROLE == 0 ? cx.stage0 : cx.stage1) + 2 * tid;   // current vector if it lives in shared memory
  const double* sn = (NEXT == 0 ? cx.stage0 : cx.stage1) + 2 * tid;   // next vector if it lives in shared memory
  const bool tail = TAIL && lim > 2 * R3_THREADS * cx.qs;  // this thread has a global tail
  const bool more = t + 1 < cx.total;
  const int i = t % cx.k;
  const int lims = cx.ncell - 2 * tid;
  const int64_t hop = P.NC - cx.ncell;
  const double* vcur = P.V[i] + (int64_t)cx.b * P.cpc + 2 * tid;                  // current vector in global memory
  const double* vnext = P.V[(t + 1) % cx.k] + (int64_t)cx.b * P.cpc + 2 * tid;     // next vector in global memory
  const unsigned long long* pollbuf = P.slots + (size_t)(t & 3) * R3_BUF_WORDS;
  unsigned long long ea0, ea1;
  r3g_poll_issue(pollbuf, cx.b, cx.G, ea0, ea1);
  if (more) {
    if (NEXT != 2 && cx.nrow > 0) mbar_wait(&sh.mbar[NEXT], (unsigned)(((t + 1) / 3) & 1), P.err);
    if (NEXT == 2) asm volatile("cp.async.wait_group 0;" ::: "memory");
    double da = 0.0, dc = 0.0;
    if (i + 1 == cx.k) {  // wrap-around into the next Gram-Schmidt pass: <v_0, v_{k-1}> is not stored, take it in the sweep
#pragma unroll
      for (int q = 0; q < R3_RP; ++q) {
        const int lr = 2 * R3_THREADS * q;  // offset from this thread's first row pair
        if (lr < lim) {
          double x0, x1, y0, y1;
          if (NEXT == 2) { R3_VRGET(q, x0, x1); }
          else if (NEXT == 0) { R3_SLOTGET(q, lr, sn, cx.stage1 + 2 * tid, TAIL && r3_dot_slot(cx, q), vnext, x0, x1); }
          else { R3_SMGET(q, lr, sn, vnext, x0, x1); }
          if (ROLE == 2) { R3_VRGET(q, y0, y1); }
          else { R3_SMGET(q, lr, sc, vcur, y0, y1); }
          da = fma(x0, w[2 * q], da); da = fma(x1, w[2 * q + 1], da);
          dc = fma(x0, y0, dc); dc = fma(x1, y1, dc);
        }
      }
      dc = warp_sum(dc);
    } else {
      double db = 0.0;  // two independent chains: 27 dependent DFMAs each instead of 54 (2 warps per scheduler cannot hide more)
#pragma unroll
      for (int q = 0; q < R3_RP; ++q) {
        const int lr = 2 * R3_THREADS * q;  // offset from this thread's first row pair
        if (lr < lim) {
          double x0, x1;
          if (NEXT == 2) { R3_VRGET(q, x0, x1); }
          else if (NEXT == 0) { R3_SLOTGET(q, lr, sn, cx.stage1 + 2 * tid, TAIL && r3_dot_slot(cx, q), vnext, x0, x1); }
          else { R3_SMGET(q, lr, sn, vnext, x0, x1); }
          da = fma(x0, w[2 * q], da); db = fma(x1, w[2 * q + 1], db);
        }
      }
      da += db;
    }
    da = warp_sum(da);
    if ((tid & 31) == 0) { sh.redA[par][tid >> 5] = da; sh.redC[par][tid >> 5] = dc; }
  }
  // Gram sub-diagonal entry <v_i, v_{i-1}>, stored when v_i was created: fetched by the spare polling thread
  if (tid == R3_SPARE_POLLER) sh.gC[par][R3_POLLERS / 32] = (i > 0) ? __ldg(P.gsub + i) : 0.0;
  r3g_poll_finish(pollbuf, cx.b, cx.G, P.epoch_base + (unsigned)t + 1u, P.err, i == 0 && t > 0, ea0, ea1, sh.gA[par], sh.gC[par]);
  // a deferred refill of stage 1 follows: its slots took the cp.async tail of v_{t+1} (completed in the sweep above); the
  // async-proxy copy into them is ordered after those writes by this fence in every writing thread and the barrier (PTX ISA,
  // memory consistency model, "Proxies": a non-bulk cp.async is a generic-proxy write, cp.async.bulk is performed in the async
  // proxy, and accesses to one location through both need a fence.proxy.async between them).  A thread that only loaded from
  // the stage needs the barrier alone, as every refill always has.
  if (ROLE == 2 && tail) fence_proxy_async_smem();
  __syncthreads();  // the only barrier of a register-role step
  if (ROLE == 2 && TAIL && t + 2 < cx.total) r3_issue_smem(P, cx, sh.mbar, t + 2, 1);
  if (more && tid < 32) {  // warp 0: total of the eight warp partials in a fixed order, then publish for step t+1
    r3_post(P.slots + (size_t)((t + 1) & 3) * R3_BUF_WORDS, cx.b, sum8(sh.redA[par]), sum8(sh.redC[par]), P.epoch_base + (unsigned)(t + 1) + 1u);
  }
  const double* gc = sh.gC[par];
  // i == 0: first vector of a pass (t == 0: nothing precedes it; t > 0: wrap-around, cross product taken in the sweep of step t-1)
  const double cross = (i > 0) ? gc[R3_POLLERS / 32] : (t > 0 ? sum5(gc) : 0.0);
  const double h = sum5(sh.gA[par]) - sh.hprev[par ^ 1] * cross;
  if (tid == 0) sh.hprev[par] = h;
  if (more) {
#pragma unroll
    for (int q = 0; q < R3_RP; ++q) {
      const int lr = 2 * R3_THREADS * q;  // offset from this thread's first row pair
      if (lr < lim) {
        double y0, y1;
        if (ROLE == 2) { R3_VRGET(q, y0, y1); }
        else { R3_SLOTGET(q, lr, sc, sc, TAIL && r3_update_slot(cx, q), vcur, y0, y1); }
        w[2 * q] = fma(-h, y0, w[2 * q]);
        w[2 * q + 1] = fma(-h, y1, w[2 * q + 1]);
      }
      if (ROLE != 2 && q + 1 == R3_TAIL_AT && cx.qs >= R3_TAIL_AT && tail) r3_tail_copy(cx, vcur, sc, R3_TAIL_AT, lim, lims, hop);
    }
  } else {  // last update of the Arnoldi step: ||w||^2 and <w, v_{k-1}> (next step's Gram sub-diagonal entry) ride along
    double nacc = 0.0, xacc = 0.0;
#pragma unroll
    for (int q = 0; q < R3_RP; ++q) {
      const int lr = 2 * R3_THREADS * q;  // offset from this thread's first row pair
      if (lr < lim) {
        double y0, y1;
        if (ROLE == 2) { R3_VRGET(q, y0, y1); }
        else { R3_SLOTGET(q, lr, sc, sc, TAIL && r3_update_slot(cx, q), vcur, y0, y1); }
        const double w0 = fma(-h, y0, w[2 * q]), w1 = fma(-h, y1, w[2 * q + 1]);
        w[2 * q] = w0; w[2 * q + 1] = w1;
        nacc = fma(w0, w0, nacc); nacc = fma(w1, w1, nacc);
        xacc = fma(w0, y0, xacc); xacc = fma(w1, y1, xacc);
      }
      if (ROLE != 2 && q + 1 == R3_TAIL_AT && cx.qs >= R3_TAIL_AT && tail) r3_tail_copy(cx, vcur, sc, R3_TAIL_AT, lim, lims, hop);
    }
    nacc = warp_sum(nacc);
    xacc = warp_sum(xacc);
    if ((tid & 31) == 0) { sh.redA[par ^ 1][tid >> 5] = nacc; sh.redC[par ^ 1][tid >> 5] = xacc; }  // parity of "step total"
  }
  if (cx.b == 0 && tid == 0) P.h[i] = (t < cx.k) ? h : P.h[i] + h;
  if (ROLE == 0 || (ROLE == 1 && !TAIL)) {
    if (t + 3 < cx.total) {
      if (tail) fence_proxy_async_smem();  // this step's cp.async tail of the stage before the bulk copy into it (see above)
      __syncthreads();                     // every thread is done with this shared-memory stage
      r3_issue_smem(P, cx, sh.mbar, t + 3, ROLE);
    }
  } else if (ROLE == 1) {  // stage 1 is refilled after the next dot sweep; until then its slots take the tail of v_{t+2}
    if (t + 3 < cx.total) r3_prefetch_l2(P, cx, t + 3);
    if (t + 2 < cx.total && tail) r3_tail_copy<false>(cx, P.V[(t + 2) % cx.k] + (int64_t)cx.b * P.cpc + 2 * tid, sc, cx.qs, lim, lims, hop);
  } else if (t + 3 < cx.total) {
    r3_issue_regs(P, cx, t + 3, vr);
  }
}

__global__ void __launch_bounds__(R3_THREADS, 1) resident3g_arnoldi_kernel(ResidentParams P) {
  if (P.st->status != 0) return;
  extern __shared__ __align__(16) double rsm[];
  __shared__ R3GShared sh;
  R3Ctx cx;
  const int cpc = P.cpc;
  const int sw = min(2 * cpc, 2 * R3_THREADS * P.qs);  // doubles per shared-memory stage
  cx.stage0 = rsm;
  cx.stage1 = rsm + sw;
  cx.annex = reinterpret_cast<double2*>(rsm + 2 * sw);
  const int tid = threadIdx.x, b = blockIdx.x, G = P.G;
  cx.b = b; cx.G = G; cx.k = P.k; cx.total = P.passes * P.k; cx.qs = P.qs;
  cx.ncell = (int)max((int64_t)0, min((int64_t)cpc, P.NC - (int64_t)b * cpc));
  cx.nrow = 2 * cx.ncell;
  if (tid == 0) {
    mbar_init(&sh.mbar[0], 1);
    mbar_init(&sh.mbar[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // the first two basis vectors start travelling while the operator is applied
  r3_issue_smem(P, cx, sh.mbar, 0, 0);
  if (cx.total > 1) r3_issue_smem(P, cx, sh.mbar, 1, 1);
  // ---- 1. w = J(u) v_k (or the assembled sparse matrix times v_k) for this CTA's rows, into registers
  double w[R3_ROWS];
  double vr[R3_VR];
  r3_apply_operator(P, cx, w);
  // ---- 2. lag-1 modified Gram-Schmidt over three rotating stages
  const int total = cx.total;
  const int nrow = cx.nrow;
  const int lim = nrow - 2 * tid;
  if (total > 2) r3_issue_regs(P, cx, 2, vr);
  {
    if (nrow > 0) mbar_wait(&sh.mbar[0], 0u, P.err);
    const int lims = cx.ncell - 2 * tid;
    const int64_t hop = P.NC - cx.ncell;
    const double* g0 = P.V[0] + (int64_t)b * cpc + 2 * tid;
    double da = 0.0;
#pragma unroll
    for (int q = 0; q < R3_RP; ++q) {
      const int lr = 2 * R3_THREADS * q;
      if (lr < lim) {
        double x0, x1;
        R3_SMGET(q, lr, cx.stage0 + 2 * tid, g0, x0, x1);
        da = fma(x0, w[2 * q], da); da = fma(x1, w[2 * q + 1], da);
      }
    }
    da = warp_sum(da);
    if ((tid & 31) == 0) sh.redA[1][tid >> 5] = da;  // parity of "step -1"
    if (tid == 0) sh.hprev[1] = 0.0;
    __syncthreads();
    if (tid < 32) r3_post(P.slots, b, sum8(sh.redA[1]), 0.0, P.epoch_base + 1u);
  }
  const bool tailed = nrow > 2 * R3_THREADS * cx.qs;
  for (int t = 0; t < total; t += 3) {
    if (tailed) {
      r3g_step<0, true>(P, cx, sh, t, w, vr);
      if (t + 1 < total) r3g_step<1, true>(P, cx, sh, t + 1, w, vr);
      if (t + 2 < total) r3g_step<2, true>(P, cx, sh, t + 2, w, vr);
    } else {
      r3g_step<0, false>(P, cx, sh, t, w, vr);
      if (t + 1 < total) r3g_step<1, false>(P, cx, sh, t + 1, w, vr);
      if (t + 2 < total) r3g_step<2, false>(P, cx, sh, t + 2, w, vr);
    }
  }
  // ---- 3. ||w|| and <w, v_{k-1}> in one exchange (the last step left the warp partials in the scratch of parity
  //         `total`), Givens (CTA 0), normalise, store v_{k+1}
  const int par = total & 1;
  __syncthreads();
  if (tid < 32) r3_post(P.slots + (size_t)(total & 3) * R3_BUF_WORDS, b, sum8(sh.redA[par]), sum8(sh.redC[par]), P.epoch_base + (unsigned)total + 1u);
  r3_poll(P.slots + (size_t)(total & 3) * R3_BUF_WORDS, b, G, P.epoch_base + (unsigned)total + 1u, P.err, sh.gA[par], sh.gC[par]);
  __syncthreads();
  const double hbis = sqrt(sum5(sh.gA[par]));
  const double inv = hbis > 0.0 ? 1.0 / hbis : 0.0;
  const int ncell = cx.ncell;
  const int64_t NC = P.NC, c0 = (int64_t)b * cpc;
#pragma unroll
  for (int q = 0; q < R3_RP; ++q) {
    const int lr = 2 * (tid + R3_THREADS * q);
    if (lr < nrow) {
      const int s = lr >= ncell;
      double2 o;
      o.x = w[2 * q] * inv; o.y = w[2 * q + 1] * inv;
      *reinterpret_cast<double2*>(P.vnew + (int64_t)s * NC + c0 + (lr - s * ncell)) = o;
    }
  }
  if (b == 0) {
    if (tid == 0) P.gsub[P.k] = sum5(sh.gC[par]) * inv;  // <v_k, v_{k-1}> for every later Arnoldi step
    resident_givens_tail(P, hbis, inv, rsm, 2 * sw, tid);
  }
}
}  // namespace

struct b200_gmres {
  b200_ctx* ctx;
  int64_t n;
  b200_gmres_opts opts;
  int G;               // CTAs of the streaming kernels
  int kcap;            // capacity (columns) of R / cs / sn / z / h / y / partial
  std::vector<double*> V;      // basis vectors (views into slabs)
  std::vector<double*> slabs;  // owning allocations
  double** d_Vptrs;
  int vptr_cap;
  double *w, *r0, *d_h, *d_hacc, *d_R, *d_cs, *d_sn, *d_z, *d_y, *d_partial, *d_norm_partial, *d_norm_partial2;
  double* d_gsub;       // resident engine: Gram sub-diagonal <v_i, v_{i-1}> (see resident3g_arnoldi_kernel)
  double* d_hraw;
  int64_t hraw_cap;
  GmresState* d_state;
  GmresState* h_state;  // pinned
  int* d_err;           // resident engine: exchange-timeout flag
  unsigned long long* d_slots;  // resident engine: four rotating exchange tables (R3_BUF_WORDS each)
  unsigned ll_epoch;
  b200_linop *Pl, *Pr;   // borrowed preconditioners (apply the inverse)
  double *pt1, *pt2;     // scratch vectors for preconditioned solves (allocated on first use)
};

namespace {
int32_t gm_free_arrays(b200_gmres* gm) {
  cudaFree(gm->d_h); cudaFree(gm->d_hacc); cudaFree(gm->d_R); cudaFree(gm->d_cs); cudaFree(gm->d_sn);
  cudaFree(gm->d_z); cudaFree(gm->d_y); cudaFree(gm->d_partial); cudaFree(gm->d_gsub);
  gm->d_h = gm->d_hacc = gm->d_R = gm->d_cs = gm->d_sn = gm->d_z = gm->d_y = gm->d_partial = gm->d_gsub = nullptr;
  return B200_OK;
}

// grow the small Krylov arrays to hold `need` columns (contents preserved)
int32_t gm_reserve(b200_gmres* gm, int need) {
  b200_ctx* ctx = gm->ctx;
  if (need <= gm->kcap) return B200_OK;
  int ncap = std::max(need, gm->kcap > 0 ? gm->kcap * 2 : 64);
  const int64_t rsz = (int64_t)ncap * (ncap + 1) / 2;
  double *nh, *nha, *nR, *ncs, *nsn, *nz, *ny, *npart, *ngs;
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (cudaMalloc(&nh, sizeof(double) * (ncap + 2)) != cudaSuccess || cudaMalloc(&nha, sizeof(double) * (ncap + 2)) != cudaSuccess ||
      cudaMalloc(&nR, sizeof(double) * rsz) != cudaSuccess || cudaMalloc(&ncs, sizeof(double) * (ncap + 2)) != cudaSuccess ||
      cudaMalloc(&nsn, sizeof(double) * (ncap + 2)) != cudaSuccess || cudaMalloc(&nz, sizeof(double) * (ncap + 2)) != cudaSuccess ||
      cudaMalloc(&ny, sizeof(double) * (ncap + 2)) != cudaSuccess || cudaMalloc(&ngs, sizeof(double) * (ncap + 2)) != cudaSuccess ||
      cudaMalloc(&npart, sizeof(double) * (int64_t)ncap * gm->G) != cudaSuccess) {
    cudaGetLastError();
    return ctx->fail(B200_ERR_NOMEM, "out of device memory growing the Krylov workspace", __FILE__, __LINE__);
  }
  if (gm->kcap > 0) {
    const int oc = gm->kcap;
    CUDA_TRY(ctx, cudaMemcpy(nR, gm->d_R, sizeof(double) * (int64_t)oc * (oc + 1) / 2, cudaMemcpyDeviceToDevice));
    CUDA_TRY(ctx, cudaMemcpy(ncs, gm->d_cs, sizeof(double) * (oc + 2), cudaMemcpyDeviceToDevice));
    CUDA_TRY(ctx, cudaMemcpy(nsn, gm->d_sn, sizeof(double) * (oc + 2), cudaMemcpyDeviceToDevice));
    CUDA_TRY(ctx, cudaMemcpy(nz, gm->d_z, sizeof(double) * (oc + 2), cudaMemcpyDeviceToDevice));
    CUDA_TRY(ctx, cudaMemcpy(ngs, gm->d_gsub, sizeof(double) * (oc + 2), cudaMemcpyDeviceToDevice));
    gm_free_arrays(gm);
  }
  gm->d_h = nh; gm->d_hacc = nha; gm->d_R = nR; gm->d_cs = ncs; gm->d_sn = nsn; gm->d_z = nz; gm->d_y = ny; gm->d_partial = npart; gm->d_gsub = ngs;
  gm->kcap = ncap;
  return B200_OK;
}

// make sure basis vectors 0..idx exist and the device pointer table covers them.  Vectors come in slabs of
// VSLAB so that growing the basis (Krylov.jl pushes new vectors past `memory` when restart = false) costs one
// allocation + one pointer-table upload per slab instead of per Arnoldi step.
constexpr int VSLAB = 16;
int32_t gm_ensure_vector(b200_gmres* gm, int idx) {
  b200_ctx* ctx = gm->ctx;
  bool table_dirty = false;
  const int64_t npad = (gm->n + 1) & ~(int64_t)1;
  while ((int)gm->V.size() <= idx) {
    double* slab = nullptr;
    int cnt = VSLAB;
    if ((int64_t)cnt * npad * 8 > ((int64_t)1 << 31)) cnt = (int)std::max<int64_t>(1, ((int64_t)1 << 31) / (npad * 8));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    if (cudaMalloc(&slab, sizeof(double) * npad * cnt) != cudaSuccess) {
      cudaGetLastError();
      cnt = 1;
      if (cudaMalloc(&slab, sizeof(double) * npad) != cudaSuccess) {
        cudaGetLastError();
        return B200_ERR_NOMEM;  // caller turns this into B200_LS_OUT_OF_MEMORY
      }
    }
    // defined contents: a kernel that early-exits on a finished status word never leaves an operand uninitialised
    CUDA_TRY(ctx, cudaMemsetAsync(slab, 0, sizeof(double) * npad * cnt, ctx->stream));
    gm->slabs.push_back(slab);
    for (int q = 0; q < cnt; ++q) gm->V.push_back(slab + (int64_t)q * npad);
    table_dirty = true;
  }
  if ((int)gm->V.size() > gm->vptr_cap) {
    int ncap = std::max((int)gm->V.size() * 2, 64);
    double** nt = nullptr;
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    CUDA_TRY(ctx, cudaMalloc(&nt, sizeof(double*) * ncap));
    if (gm->d_Vptrs) cudaFree(gm->d_Vptrs);
    gm->d_Vptrs = nt;
    gm->vptr_cap = ncap;
    table_dirty = true;
  }
  if (table_dirty) {
    CUDA_TRY(ctx, cudaMemcpyAsync(gm->d_Vptrs, gm->V.data(), sizeof(double*) * gm->V.size(), cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  }
  return B200_OK;
}

int32_t gm_fetch_state(b200_gmres* gm) {
  b200_ctx* ctx = gm->ctx;
  CUDA_TRY(ctx, cudaMemcpyAsync(gm->h_state, gm->d_state, sizeof(GmresState), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return B200_OK;
}
}  // namespace

// ------------------------------------------------------------------ operator application (K2/K3)
namespace {
// y = D^-1 x, D = the 2x2 species blocks on the diagonal of the Brusselator Jacobian at u (cell c couples rows c and NC + c)
__global__ void __launch_bounds__(GM_THREADS) block_jacobi_kernel(int64_t NC, double lapdiag, double A, const double* __restrict__ u, const double* __restrict__ x,
                                                                   double* __restrict__ y) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= NC) return;
  const double uc = u[c], vc = u[c + NC];
  const double d00 = lapdiag + (2.0 * uc * vc - (A + 1.0)), d01 = uc * uc, d10 = A - 2.0 * uc * vc, d11 = lapdiag - uc * uc;
  const double det = d00 * d11 - d01 * d10;
  const double x0 = x[c], x1 = x[c + NC];
  y[c] = (d11 * x0 - d01 * x1) / det;
  y[c + NC] = (d00 * x1 - d10 * x0) / det;
}
}  // namespace

static int32_t linop_apply_unshifted(b200_linop* op, const double* x, double* y);
int32_t b200i_linop_apply(b200_linop* op, const double* x, double* y) {
  B200_TRY(linop_apply_unshifted(op, x, y));
  if (op->shift != 0.0) B200_TRY(b200_axpy(op->ctx, op->n, op->shift, x, y));
  return B200_OK;
}
static int32_t linop_apply_unshifted(b200_linop* op, const double* x, double* y) {
  b200_ctx* ctx = op->ctx;
  switch (op->kind) {
    case LINOP_PROBLEM:
      return op->jvp_mode == B200_JVP_FINITE_DIFF ? b200_jvp_fd(op->prob, op->u, x, y) : b200_jvp(op->prob, op->u, x, y);
    case LINOP_CSC: {
      LAUNCH(ctx, csc_rows_spmv_kernel, (int)((op->n + GM_THREADS - 1) / GM_THREADS), GM_THREADS, 0, op->n, (const int64_t*)op->csr_rowptr,
             (const int64_t*)op->csr_col, (const int64_t*)op->csr_map, op->nzval, x, y);
      CHECK_LAUNCH(ctx);
      return B200_OK;
    }
    case LINOP_DENSE:
      return b200_gemv(ctx, 0, op->n, op->n, op->A, op->ld, x, y);
    case LINOP_CALLBACK:
      B200_TRY(b200i_sync_for_callback(ctx));
      return op->mv(op->user, x, y) == 0 ? B200_OK : ctx->fail(B200_ERR_CALLBACK, "matvec callback failed", __FILE__, __LINE__);
    case LINOP_SPARSE_JAC:
      return b200_spmv(op->sj, op->nzval, x, y);
    case LINOP_MULTIGRID:
      return b200i_mg_apply(op->mg, x, y);
    case LINOP_ILU0:
      return b200_ilu0_solve(op->ilu, x, y);
    case LINOP_AMG:
      return b200_amg_solve(op->amg, x, y);
    case LINOP_BLOCK_JACOBI: {
      const int64_t NC = op->n / 2;
      const double lapdiag = -(op->prob->kind == B200_PROB_BRUSS3D ? 6.0 : 4.0) * op->prob->a;
      LAUNCH(ctx, block_jacobi_kernel, (int)((NC + GM_THREADS - 1) / GM_THREADS), GM_THREADS, 0, NC, lapdiag, op->prob->A, op->u, x, y);
      CHECK_LAUNCH(ctx);
      return B200_OK;
    }
  }
  return ctx->fail(B200_ERR_INVALID, "unknown linop kind", __FILE__, __LINE__);
}

// ------------------------------------------------------------------ resident engine (host side)
namespace {
struct ResidentPlan {
  ResidentParams base;  // the step-independent fields: operator, geometry, passes
  size_t smem;          // dynamic shared memory of resident3g_arnoldi_kernel: two stages + the annex of the register stage
};

// raw Hessenberg column k of a capture (b200_gmres_keep_hessenberg), or null when there is none or it is full
double* gm_hraw(const b200_gmres* gm, int k) { return (gm->d_hraw && (int64_t)k * (k + 3) / 2 <= gm->hraw_cap) ? gm->d_hraw : nullptr; }

// algorithmic bytes of resident Arnoldi step k: the basis once per pass + u, v_k reads + v_{k+1} store
double resident_step_bytes(int passes, int k, double Bv) { return (passes * (double)k + 3.0) * Bv; }

// Decides whether this solve runs on the resident engine (*use) and, if so, its plan.  Built-in Brusselator operator with the
// exact JVP (or an assembled sparse Jacobian), even cell count, one CTA per SM holds its rows: <= 60 rows per thread; the
// register stage's annex and at least one row pair per thread of each shared-memory stage must fit (the stages hold as many
// pairs as the shared memory left beside the annex takes).  engine = resident fails when any of that does not hold.
// tests/test_gpu_resident_geometry.py restates this selection independently (its `Geometry` class).
int32_t gm_resident_plan(b200_gmres* gm, b200_linop* op, bool* use, ResidentPlan* plan) {
  b200_ctx* ctx = gm->ctx;
  const b200_gmres_opts& o = gm->opts;
  const int64_t n = gm->n;
  *use = false;
  memset(plan, 0, sizeof(*plan));
  const bool builtin = op->kind == LINOP_PROBLEM && op->jvp_mode == B200_JVP_EXACT && (op->prob->kind == B200_PROB_BRUSS2D || op->prob->kind == B200_PROB_BRUSS3D);
  const bool csr = op->kind == LINOP_SPARSE_JAC && n % 2 == 0;
  const bool precond = gm->Pl || gm->Pr;
  if (precond && o.engine == B200_ENGINE_RESIDENT)
    return ctx->fail(B200_ERR_UNSUPPORTED, "resident GMRES engine does not take preconditioners (use engine = auto / multikernel)", __FILE__, __LINE__);
  if (op->shift != 0.0 && o.engine == B200_ENGINE_RESIDENT)
    return ctx->fail(B200_ERR_UNSUPPORTED, "resident GMRES engine does not take shifted operators (use engine = auto / multikernel)", __FILE__, __LINE__);
  if (o.engine == B200_ENGINE_MULTIKERNEL || !(builtin || csr) || precond || op->shift != 0.0) {
    if (o.engine == B200_ENGINE_RESIDENT)
      return ctx->fail(B200_ERR_UNSUPPORTED, "resident GMRES engine needs a built-in Brusselator operator with the exact JVP or an assembled sparse Jacobian", __FILE__, __LINE__);
    return B200_OK;
  }
  ResidentParams& RP = plan->base;
  RP.passes = (o.orth == B200_ORTH_CGS2) ? 2 : 1;
  RP.NC = n / 2;
  RP.G = ctx->sm_count;
  int64_t cpc = (RP.NC + RP.G - 1) / RP.G;
  cpc = (cpc + 1) & ~(int64_t)1;
  RP.cpc = (int)cpc;
  const size_t pair_bytes = 2 * sizeof(double) * 2 * R3_THREADS;  // one row pair per thread in both stages
  const size_t spare = ctx->smem_optin > R3_ANNEX_BYTES + 2048 ? ctx->smem_optin - R3_ANNEX_BYTES - 2048 : 0;
  RP.qs = (int)std::min<int64_t>(std::min<int64_t>(R3_RP, (2 * cpc + 2 * R3_THREADS - 1) / (2 * R3_THREADS)), (int64_t)(spare / pair_bytes));
  // diagnostic: cap the stages at fewer row pairs per thread, so that rows move to the global-memory tail (same arithmetic)
  static_assert(R3_RP == 30, "the message below states the range");
  if (const char* e = getenv("B200_RESIDENT_STAGE_PAIRS")) {
    char* end = nullptr;
    const long cap = strtol(e, &end, 10);
    if (end == e || *end != '\0' || cap < 1 || cap > R3_RP)
      return ctx->fail(B200_ERR_INVALID, "B200_RESIDENT_STAGE_PAIRS must be an integer in 1..30 (row pairs per thread of the resident engine's shared-memory stages)", __FILE__, __LINE__);
    RP.qs = std::min(RP.qs, (int)cap);
  }
  const int64_t stage_words = std::min<int64_t>(2 * cpc, (int64_t)2 * R3_THREADS * RP.qs);
  plan->smem = sizeof(double) * 2 * (size_t)stage_words + R3_ANNEX_BYTES;
  const bool fits = (RP.NC % 2 == 0) && RP.G <= R3_SPARE_POLLER && (2 * cpc <= (int64_t)R3_ROWS * R3_THREADS) && RP.qs >= 1;
  const bool wanted = (o.engine == B200_ENGINE_RESIDENT) || (o.engine == B200_ENGINE_AUTO && n >= 200000);
  if (!fits || !wanted) {
    if (o.engine == B200_ENGINE_RESIDENT)
      return ctx->fail(B200_ERR_UNSUPPORTED, "resident GMRES engine: problem does not fit (needs an even cell count and at most 7680 cells per SM)", __FILE__, __LINE__);
    return B200_OK;
  }
  if (csr) {
    RP.opkind = 1;
    b200i_sparse_jac_csr(op->sj, &RP.rowptr, &RP.csr_col, &RP.csr_map);
    RP.nzval = op->nzval;
  } else {
    RP.dim = op->prob->kind == B200_PROB_BRUSS2D ? 2 : 3;
    RP.N = op->prob->N; RP.a = op->prob->a; RP.A = op->prob->A; RP.u = op->u;
  }
  CUDA_TRY(ctx, cudaFuncSetAttribute(resident3g_arnoldi_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)plan->smem));
  *use = true;
  return B200_OK;
}

// Arnoldi step k on the resident engine: one cooperative kernel, JVP -> (iterated) MGS with TMA-staged basis -> norm -> Givens -> v_{k+1}
int32_t gm_resident_step(b200_gmres* gm, const ResidentPlan& plan, int k) {
  b200_ctx* ctx = gm->ctx;
  ResidentParams RP = plan.base;
  RP.k = k;
  RP.V = (const double* const*)gm->d_Vptrs; RP.vnew = gm->V[k];
  if (gm->ll_epoch > 0xfff00000u) {  // epoch space nearly exhausted: start over with clean slots
    CUDA_TRY(ctx, cudaMemsetAsync(gm->d_slots, 0, sizeof(unsigned long long) * 4 * R3_BUF_WORDS, ctx->stream));
    gm->ll_epoch = 0;
  }
  RP.slots = gm->d_slots; RP.epoch_base = gm->ll_epoch; RP.err = gm->d_err;
  gm->ll_epoch += (unsigned)(RP.passes * k + 2);
  RP.h = gm->d_h; RP.gsub = gm->d_gsub; RP.R = gm->d_R; RP.cs = gm->d_cs; RP.sn = gm->d_sn; RP.z = gm->d_z;
  RP.hraw = gm_hraw(gm, k);
  RP.st = gm->d_state;
  return coop_launch(ctx, B200_KID_RESIDENT, resident_step_bytes(RP.passes, k, 8.0 * (double)gm->n), resident3g_arnoldi_kernel, RP.G, R3_THREADS, plan.smem,
                     RP);
}
}  // namespace

extern "C" {
int32_t b200_gemv(b200_ctx* ctx, int32_t trans, int64_t m, int64_t n, const double* A, int64_t ld, const double* x, double* y) {
  B200_DEVICE_GUARD(ctx);
  if (!trans) {
    LAUNCH(ctx, dense_gemv_kernel, (int)((m + GM_THREADS - 1) / GM_THREADS), GM_THREADS, 0, 0, m, n, A, ld, x, y);
  } else if (n <= 64 && m >= 32768) {  // tall and skinny: all columns in one pass over the rows, TG_NC columns at a time
    const int G = (int)std::min<int64_t>(512, (m + 4095) / 4096);
    for (int64_t c0 = 0; c0 < n; c0 += TG_NC) {
      const int nc = (int)std::min<int64_t>(TG_NC, n - c0);
      LAUNCH(ctx, tall_gemvt_partial_kernel, G, GM_THREADS, 0, m, nc, A + c0 * ld, ld, x, ctx->d_partials);
      LAUNCH(ctx, tall_gemvt_final_kernel, 1, 32, 0, nc, G, (const double*)ctx->d_partials, y + c0);
    }
  } else {
    LAUNCH(ctx, dense_gemv_kernel, (int)std::min<int64_t>(n, 4096), GM_THREADS, 0, 1, m, n, A, ld, x, y);
  }
  CHECK_LAUNCH(ctx);
  return B200_OK;
}

int32_t b200_linop_from_problem(b200_problem* prob, const double* u, int32_t jvp_mode, b200_linop** out) {
  B200_DEVICE_GUARD(prob ? prob->ctx : nullptr);
  b200_linop* op = new b200_linop();
  memset(op, 0, sizeof(*op));
  op->ctx = prob->ctx; op->kind = LINOP_PROBLEM; op->n = prob->n; op->prob = prob; op->u = u; op->jvp_mode = jvp_mode;
  *out = op;
  return B200_OK;
}
int32_t b200_linop_from_csc(b200_ctx* ctx, int64_t n, const int64_t* colptr, const int64_t* rowval, const double* nzval, int32_t base,
                            b200_linop** out) {
  B200_DEVICE_GUARD(ctx);
  B200_REQUIRE(ctx, n > 0 && colptr && rowval && nzval && out, "linop_from_csc: bad arguments");
  // row view of the pattern, built once on the host (index arrays only; the values stay where they are and may change)
  std::vector<int64_t> cp(n + 1);
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  CUDA_TRY(ctx, cudaMemcpy(cp.data(), colptr, sizeof(int64_t) * (n + 1), cudaMemcpyDeviceToHost));
  const int64_t nnz = cp[n] - base;
  B200_REQUIRE(ctx, nnz >= 0, "linop_from_csc: colptr is not a CSC column pointer with this index_base");
  std::vector<int64_t> rv((size_t)std::max<int64_t>(nnz, 1)), rowptr(n + 1, 0), ccol((size_t)std::max<int64_t>(nnz, 1)), cmap((size_t)std::max<int64_t>(nnz, 1));
  if (nnz > 0) CUDA_TRY(ctx, cudaMemcpy(rv.data(), rowval, sizeof(int64_t) * nnz, cudaMemcpyDeviceToHost));
  for (int64_t k = 0; k < nnz; ++k) {
    const int64_t r = rv[k] - base;
    if (r < 0 || r >= n) return ctx->fail(B200_ERR_INVALID, "linop_from_csc: row index out of range", __FILE__, __LINE__);
    rowptr[r + 1]++;
  }
  for (int64_t r = 0; r < n; ++r) rowptr[r + 1] += rowptr[r];
  {
    std::vector<int64_t> fill(rowptr.begin(), rowptr.end() - 1);
    for (int64_t c = 0; c < n; ++c)
      for (int64_t k = cp[c] - base; k < cp[c + 1] - base; ++k) { const int64_t q = fill[rv[k] - base]++; ccol[q] = c; cmap[q] = k; }
  }
  b200_linop* op = new b200_linop();
  memset(op, 0, sizeof(*op));
  op->ctx = ctx; op->kind = LINOP_CSC; op->n = n; op->colptr = colptr; op->rowval = rowval; op->nzval = nzval; op->index_base = base;
  bool ok = cudaMalloc(&op->csr_rowptr, sizeof(int64_t) * (n + 1)) == cudaSuccess && cudaMalloc(&op->csr_col, sizeof(int64_t) * std::max<int64_t>(nnz, 1)) == cudaSuccess &&
            cudaMalloc(&op->csr_map, sizeof(int64_t) * std::max<int64_t>(nnz, 1)) == cudaSuccess;
  if (ok) ok = cudaMemcpy(op->csr_rowptr, rowptr.data(), sizeof(int64_t) * (n + 1), cudaMemcpyHostToDevice) == cudaSuccess &&
               cudaMemcpy(op->csr_col, ccol.data(), sizeof(int64_t) * nnz, cudaMemcpyHostToDevice) == cudaSuccess &&
               cudaMemcpy(op->csr_map, cmap.data(), sizeof(int64_t) * nnz, cudaMemcpyHostToDevice) == cudaSuccess;
  if (!ok) {
    cudaGetLastError();
    cudaFree(op->csr_rowptr); cudaFree(op->csr_col); cudaFree(op->csr_map);
    delete op;
    return ctx->fail(B200_ERR_NOMEM, "linop_from_csc: cannot allocate the row view", __FILE__, __LINE__);
  }
  *out = op;
  return B200_OK;
}
int32_t b200_linop_from_dense(b200_ctx* ctx, int64_t n, const double* A, int64_t ld, b200_linop** out) {
  B200_DEVICE_GUARD(ctx);
  b200_linop* op = new b200_linop();
  memset(op, 0, sizeof(*op));
  op->ctx = ctx; op->kind = LINOP_DENSE; op->n = n; op->A = A; op->ld = ld;
  *out = op;
  return B200_OK;
}
int32_t b200_linop_from_callback(b200_ctx* ctx, int64_t n, b200_matvec_cb mv, void* user, b200_linop** out) {
  B200_DEVICE_GUARD(ctx);
  b200_linop* op = new b200_linop();
  memset(op, 0, sizeof(*op));
  op->ctx = ctx; op->kind = LINOP_CALLBACK; op->n = n; op->mv = mv; op->user = user;
  *out = op;
  return B200_OK;
}
int32_t b200_linop_apply(b200_linop* op, const double* x, double* y) {
  B200_DEVICE_GUARD(op ? op->ctx : nullptr);
  return b200i_linop_apply(op, x, y);
}
int32_t b200_linop_set_shift(b200_linop* op, double shift) { op->shift = shift; return B200_OK; }
int32_t b200_linop_destroy(b200_linop* op) {
  if (!op) return B200_OK;
  B200_DEVICE_GUARD(op->ctx);
  if (op->mg && op->owns_mg) b200i_mg_destroy(op->mg);
  if (op->csr_rowptr) { cudaStreamSynchronize(op->ctx->stream); cudaFree(op->csr_rowptr); cudaFree(op->csr_col); cudaFree(op->csr_map); }
  delete op;
  return B200_OK;
}

void b200_gmres_opts_default(b200_gmres_opts* o) {
  memset(o, 0, sizeof(*o));
  o->memory = 20;        // Krylov.jl default `memory`; LinearSolve passes min(20, n)
  o->restart = 0;        // KrylovJL_GMRES(gmres_restart = 0): no restart
  o->itmax = 0;          // => n
  o->orth = B200_ORTH_CGS2;
  o->warm_start = 0;
  o->engine = B200_ENGINE_AUTO;
  o->check_every = 0;  // 0 => 8, or 2 when a preconditioner is attached (see b200_gmres_solve)
  o->atol = 0.0;
  o->rtol = 1.4901161193847656e-08;  // sqrt(eps): Krylov.jl default rtol
}

int32_t b200_gmres_create(b200_ctx* ctx, int64_t n, const b200_gmres_opts* opts, b200_gmres** out) {
  B200_DEVICE_GUARD(ctx);
  B200_REQUIRE(ctx, n > 0 && opts && out, "gmres_create: bad arguments");
  b200_gmres* gm = new b200_gmres();
  gm->ctx = ctx; gm->n = n; gm->opts = *opts;
  gm->kcap = 0; gm->d_Vptrs = nullptr; gm->vptr_cap = 0;
  gm->d_h = gm->d_hacc = gm->d_R = gm->d_cs = gm->d_sn = gm->d_z = gm->d_y = gm->d_partial = gm->d_gsub = nullptr;
  gm->d_hraw = nullptr; gm->hraw_cap = 0;
  gm->d_err = nullptr; gm->d_slots = nullptr; gm->ll_epoch = 0; gm->Pl = gm->Pr = nullptr; gm->pt1 = gm->pt2 = nullptr;
  // streaming grid: 4 CTAs of 256 threads per SM, fewer for small n (at least 512 rows per CTA)
  int64_t g = std::min<int64_t>((int64_t)ctx->sm_count * 4, std::max<int64_t>(1, n / 512));
  gm->G = (int)g;
  const int64_t npad = (n + 1) & ~(int64_t)1;
  CUDA_TRY(ctx, cudaMalloc(&gm->w, sizeof(double) * npad));
  CUDA_TRY(ctx, cudaMalloc(&gm->r0, sizeof(double) * npad));
  CUDA_TRY(ctx, cudaMalloc(&gm->d_norm_partial, sizeof(double) * std::max(gm->G, B200_RED_MAX_BLOCKS)));
  CUDA_TRY(ctx, cudaMalloc(&gm->d_norm_partial2, sizeof(double) * std::max(gm->G, B200_RED_MAX_BLOCKS)));
  CUDA_TRY(ctx, cudaMalloc(&gm->d_state, sizeof(GmresState)));
  CUDA_TRY(ctx, cudaMallocHost(&gm->h_state, sizeof(GmresState)));
  CUDA_TRY(ctx, cudaMalloc(&gm->d_err, sizeof(int)));
  CUDA_TRY(ctx, cudaMalloc(&gm->d_slots, sizeof(unsigned long long) * 4 * R3_BUF_WORDS));
  CUDA_TRY(ctx, cudaMemsetAsync(gm->d_slots, 0, sizeof(unsigned long long) * 4 * R3_BUF_WORDS, ctx->stream));
  CUDA_TRY(ctx, cudaMemsetAsync(gm->d_err, 0, sizeof(int), ctx->stream));
  CUDA_TRY(ctx, cudaFuncSetAttribute(update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(double) * (GM_KCAP + 64))));
  CUDA_TRY(ctx, cudaFuncSetAttribute(backsolve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(double) * (GM_KCAP + 64))));
  int mem = opts->restart > 0 ? opts->restart : (opts->memory > 0 ? opts->memory : 20);
  if (mem > n) mem = (int)n;
  int32_t s = gm_reserve(gm, std::max(mem + 1, 32));
  if (s != B200_OK) { b200_gmres_destroy(gm); return s; }
  *out = gm;
  return B200_OK;
}

int32_t b200_gmres_destroy(b200_gmres* gm) {
  B200_DEVICE_GUARD(gm ? gm->ctx : nullptr);
  if (!gm) return B200_OK;
  cudaStreamSynchronize(gm->ctx->stream);
  for (double* v : gm->slabs) cudaFree(v);
  if (gm->d_Vptrs) cudaFree(gm->d_Vptrs);
  cudaFree(gm->w); cudaFree(gm->r0); cudaFree(gm->d_norm_partial); cudaFree(gm->d_norm_partial2); cudaFree(gm->d_state);
  if (gm->d_hraw) cudaFree(gm->d_hraw);
  cudaFreeHost(gm->h_state);
  if (gm->d_err) cudaFree(gm->d_err);
  if (gm->d_slots) cudaFree(gm->d_slots);
  if (gm->pt1) cudaFree(gm->pt1);
  if (gm->pt2) cudaFree(gm->pt2);
  gm_free_arrays(gm);
  delete gm;
  return B200_OK;
}

int32_t b200_gmres_set_tolerances(b200_gmres* gm, double atol, double rtol) {
  if (atol >= 0) gm->opts.atol = atol;
  if (rtol >= 0) gm->opts.rtol = rtol;
  return B200_OK;
}
int32_t b200_gmres_set_precond(b200_gmres* gm, b200_linop* left_inv, b200_linop* right_inv) {
  B200_DEVICE_GUARD(gm ? gm->ctx : nullptr);
  b200_ctx* ctx = gm->ctx;
  B200_REQUIRE(ctx, (!left_inv || left_inv->n == gm->n) && (!right_inv || right_inv->n == gm->n), "gmres_set_precond: operator size mismatch");
  gm->Pl = left_inv; gm->Pr = right_inv;
  if ((left_inv || right_inv) && !gm->pt1) {
    CUDA_TRY(ctx, cudaMalloc(&gm->pt1, sizeof(double) * (gm->n + 2)));
    CUDA_TRY(ctx, cudaMalloc(&gm->pt2, sizeof(double) * (gm->n + 2)));
  }
  return B200_OK;
}
int32_t b200_linop_block_jacobi(b200_problem* prob, const double* u, b200_linop** out) {
  B200_DEVICE_GUARD(prob ? prob->ctx : nullptr);
  B200_REQUIRE(prob->ctx, prob->kind == B200_PROB_BRUSS2D || prob->kind == B200_PROB_BRUSS3D, "block-Jacobi preconditioner: built-in Brusselator problems only");
  b200_linop* op = new b200_linop();
  memset(op, 0, sizeof(*op));
  op->ctx = prob->ctx; op->kind = LINOP_BLOCK_JACOBI; op->n = prob->n; op->prob = prob; op->u = u;
  *out = op;
  return B200_OK;
}

int32_t b200_linop_precond(b200_problem* prob, const double* u, int32_t kind, b200_linop** out) {
  B200_DEVICE_GUARD(prob ? prob->ctx : nullptr);
  b200_ctx* ctx = prob->ctx;
  B200_REQUIRE(ctx, u && out, "linop_precond: bad arguments");
  if (kind == B200_PRECOND_BLOCK_JACOBI_LEFT || kind == B200_PRECOND_BLOCK_JACOBI_RIGHT) return b200_linop_block_jacobi(prob, u, out);
  B200_REQUIRE(ctx, kind != B200_PRECOND_ILU0_LEFT && kind != B200_PRECOND_ILU0_RIGHT,
               "linop_precond: ILU0 factors the assembled sparse Jacobian, not a problem: use b200_ilu0_create / b200_ilu0_factor / b200_ilu0_linop");
  B200_REQUIRE(ctx, kind != B200_PRECOND_AMG_LEFT && kind != B200_PRECOND_AMG_RIGHT && kind != B200_PRECOND_SA_AMG_LEFT && kind != B200_PRECOND_SA_AMG_RIGHT,
               "linop_precond: AMG coarsens the assembled sparse Jacobian, not a problem: use b200_amg_create (or b200_amg_create_sa) / b200_amg_setup / b200_amg_linop");
  B200_REQUIRE(ctx, kind == B200_PRECOND_MULTIGRID_LEFT || kind == B200_PRECOND_MULTIGRID_RIGHT, "linop_precond: unknown preconditioner kind");
  b200_mg* mg = nullptr;
  B200_TRY(b200i_mg_create(prob, &mg));
  int32_t st = b200i_mg_setup(mg, u);
  if (st != B200_OK) { b200i_mg_destroy(mg); return st; }
  b200_linop* op = new b200_linop();
  memset(op, 0, sizeof(*op));
  op->ctx = ctx; op->kind = LINOP_MULTIGRID; op->n = prob->n; op->prob = prob; op->u = u; op->mg = mg; op->owns_mg = 1;
  *out = op;
  return B200_OK;
}

// test hook: keep the raw Hessenberg columns of the next solve (k+1 entries per column)
int32_t b200_gmres_keep_hessenberg(b200_gmres* gm, int64_t capacity) {
  B200_DEVICE_GUARD(gm ? gm->ctx : nullptr);
  b200_ctx* ctx = gm->ctx;
  if (gm->d_hraw) { cudaFree(gm->d_hraw); gm->d_hraw = nullptr; }
  gm->hraw_cap = capacity;
  if (capacity > 0) CUDA_TRY(ctx, cudaMalloc(&gm->d_hraw, sizeof(double) * capacity));
  return B200_OK;
}
int32_t b200_gmres_get_hessenberg(b200_gmres* gm, double* out_host, int64_t count) {
  B200_DEVICE_GUARD(gm ? gm->ctx : nullptr);
  b200_ctx* ctx = gm->ctx;
  if (!gm->d_hraw || count > gm->hraw_cap) return ctx->fail(B200_ERR_INVALID, "hessenberg capture not enabled / too small", __FILE__, __LINE__);
  return b200_memcpy_d2h(ctx, out_host, gm->d_hraw, sizeof(double) * count);
}

int32_t b200_gmres_solve(b200_gmres* gm, b200_linop* op, const double* b, double* x, b200_gmres_stats* stats) {
  B200_DEVICE_GUARD(gm ? gm->ctx : nullptr);
  b200_ctx* ctx = gm->ctx;
  B200_REQUIRE(ctx, op && op->n == gm->n && b && x, "gmres_solve: bad arguments");
  B200_REQUIRE(ctx, (reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(b) & 7) == 0,
               "gmres_solve: x must be 16-byte aligned (vectorised loads)");
  const int64_t n = gm->n;
  const b200_gmres_opts& o = gm->opts;
  const int G = gm->G;
  const int orth = o.orth;
  // operators that run host code between kernels (callbacks; preconditioners synchronise per apply anyway) must never be
  // handed the operand of an iteration that a finished solve skipped: poll the device status every iteration for them
  const bool host_op = op->kind == LINOP_CALLBACK || (op->kind == LINOP_PROBLEM && op->prob->kind == B200_PROB_CALLBACK) ||
                       (gm->Pl && gm->Pl->kind == LINOP_CALLBACK) || (gm->Pr && gm->Pr->kind == LINOP_CALLBACK);
  // with a preconditioner an iteration is expensive (a V-cycle per step) and the basis short: iterations enqueued after
  // convergence still run the preconditioner's kernels, so the status is polled every other step (default 8 otherwise)
  const int check_every = host_op ? 1 : (o.check_every > 0 ? o.check_every : ((gm->Pl || gm->Pr) ? 2 : 8));
  b200_linop *Pl = gm->Pl, *Pr = gm->Pr;
  bool resident = false;
  ResidentPlan rs;
  B200_TRY(gm_resident_plan(gm, op, &resident, &rs));
  const int64_t itmax = o.itmax > 0 ? o.itmax : n;
  const int restart_len = o.restart > 0 ? (int)std::min<int64_t>(o.restart, n) : 0;
  const int ew_grid = (int)std::min<int64_t>((n + GM_THREADS * 2 - 1) / (GM_THREADS * 2), (int64_t)ctx->sm_count * 8);
  b200_gmres_stats st_local;
  memset(&st_local, 0, sizeof(st_local));
  double bytes = 0.0;
  const double Bv = 8.0 * (double)n;

  // ---- initial state
  GmresState init;
  memset(&init, 0, sizeof(init));
  init.itmax = (int32_t)std::min<int64_t>(itmax, INT32_MAX);
  init.kmax_cycle = restart_len > 0 ? restart_len : INT32_MAX;
  init.atol = o.atol;
  init.rtol = o.rtol;
  *gm->h_state = init;
  CUDA_TRY(ctx, cudaMemsetAsync(gm->d_err, 0, sizeof(int), ctx->stream));  // resident engine: exchange-timeout flag of a previous solve
  CUDA_TRY(ctx, cudaMemcpyAsync(gm->d_state, gm->h_state, sizeof(GmresState), cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));  // h_state is reused as the read-back buffer below

  int32_t rc = gm_ensure_vector(gm, 1);
  if (rc == B200_ERR_NOMEM) return ctx->fail(B200_ERR_NOMEM, "cannot allocate the first Krylov vectors", __FILE__, __LINE__);
  B200_TRY(rc);

  int nmatvec = 0, restarts = 0;
  int64_t iters_total = 0;
  bool first_cycle = true;
  bool have_x = o.warm_start != 0;
  if (!have_x) CUDA_TRY(ctx, cudaMemsetAsync(x, 0, sizeof(double) * n, ctx->stream));
  int final_status = 0;
  int oom = 0;

  for (;;) {
    // r0 = b - A x (or b), beta, V[0] = r0 / beta
    const double* Ax = nullptr;
    if (have_x) {
      B200_TRY(b200i_linop_apply(op, x, gm->w));
      ++nmatvec;
      Ax = gm->w;
      bytes += 3 * Bv;
    }
    LAUNCH(ctx, residual_init_kernel, std::min(G, B200_RED_MAX_BLOCKS), GM_THREADS, 0, n, b, Ax, gm->r0, gm->d_norm_partial);
    if (Pl) {  // r0 <- M^-1 (b - A x): the iteration and its stopping test live in the left-preconditioned space
      B200_TRY(b200i_linop_apply(Pl, gm->r0, gm->pt1));
      LAUNCH(ctx, residual_init_kernel, std::min(G, B200_RED_MAX_BLOCKS), GM_THREADS, 0, n, (const double*)gm->pt1, (const double*)nullptr, gm->r0, gm->d_norm_partial);
      bytes += 5 * Bv;
    }
    LAUNCH(ctx, init_finish_kernel, 1, GM_THREADS, 0, gm->d_state, std::min(G, B200_RED_MAX_BLOCKS), gm->d_norm_partial, gm->d_z,
           first_cycle ? 1 : 0);
    LAUNCH(ctx, normalize_kernel, ew_grid, GM_THREADS, 0, gm->d_state, 0, gm->r0, gm->V[0], n);
    CHECK_LAUNCH(ctx);
    bytes += (Ax ? 3 : 2) * Bv + 2 * Bv;
    first_cycle = false;

    int k = 0;
    int cycle_status = 0;
    if (host_op) {  // ||r0|| <= tol (or a non-finite start): do not call user code at all
      B200_TRY(gm_fetch_state(gm));
      cycle_status = gm->h_state->status;
    }
    while (cycle_status == 0) {
      ++k;
      B200_TRY(gm_reserve(gm, k + 1));
      rc = gm_ensure_vector(gm, k);
      // The basis cannot grow any further (device memory, or the GM_KCAP coefficients the update / back-substitution
      // kernels stage in shared memory): Krylov.jl would keep going up to itmax = n; the closest thing that still
      // converges is an implicit restart from the current iterate.  Only a basis too small to be useful is a failure.
      if (rc == B200_ERR_NOMEM || k + 40 > GM_KCAP) { oom = 1; --k; break; }
      B200_TRY(rc);
      if (resident) {
        B200_TRY(gm_resident_step(gm, rs, k));
      } else {
        // w = M^-1 A N^-1 v_k
        const double* in = gm->V[k - 1];
        if (Pr) { B200_TRY(b200i_linop_apply(Pr, in, gm->pt1)); in = gm->pt1; bytes += 3 * Bv; }
        if (Pl) {
          B200_TRY(b200i_linop_apply(op, in, gm->pt2));
          B200_TRY(b200i_linop_apply(Pl, gm->pt2, gm->w));
          bytes += 3 * Bv;
        } else {
          B200_TRY(b200i_linop_apply(op, in, gm->w));
        }
        const double* norm_partial = gm->d_norm_partial;
        if (orth == B200_ORTH_MGS) {
          double* pin = gm->d_norm_partial;
          double* pout = gm->d_norm_partial2;
          PLAUNCH(ctx, B200_KID_MGS, 2.0 * Bv, mgs_pass_kernel, G, GM_THREADS, 0, gm->d_state, (const double*)nullptr, (const double*)gm->V[0], -1, pin, pout, gm->d_h,
                  gm->w, n);
          for (int i = 0; i < k; ++i) {
            std::swap(pin, pout);
            PLAUNCH(ctx, B200_KID_MGS, 4.0 * Bv, mgs_pass_kernel, G, GM_THREADS, 0, gm->d_state, (const double*)gm->V[i],
                    (const double*)(i + 1 < k ? gm->V[i + 1] : nullptr), i, pin, pout, gm->d_h, gm->w, n);
          }
          norm_partial = pout;
        } else {
          const size_t shm = sizeof(double) * (k + 32);
          PLAUNCH(ctx, B200_KID_MULTIDOT, (k + 1.0) * Bv, multidot_kernel, G, GM_THREADS, 0, gm->d_state, (const double* const*)gm->d_Vptrs, k, gm->w, n, gm->d_partial);
          LAUNCH(ctx, reduce_h_kernel, (k + 7) / 8, GM_THREADS, 0, gm->d_state, k, G, gm->d_partial, gm->d_h, (double*)nullptr);
          PLAUNCH(ctx, B200_KID_UPDATE, (k + 2.0) * Bv, update_kernel, G, GM_THREADS, shm, gm->d_state, 0, (const double* const*)gm->d_Vptrs, k, gm->d_h, -1.0, gm->w, gm->w, n,
                  gm->d_norm_partial);
          if (orth == B200_ORTH_CGS2) {
            PLAUNCH(ctx, B200_KID_MULTIDOT, (k + 1.0) * Bv, multidot_kernel, G, GM_THREADS, 0, gm->d_state, (const double* const*)gm->d_Vptrs, k, gm->w, n, gm->d_partial);
            LAUNCH(ctx, reduce_h_kernel, (k + 7) / 8, GM_THREADS, 0, gm->d_state, k, G, gm->d_partial, gm->d_hacc, gm->d_h);
            PLAUNCH(ctx, B200_KID_UPDATE, (k + 2.0) * Bv, update_kernel, G, GM_THREADS, shm, gm->d_state, 0, (const double* const*)gm->d_Vptrs, k, gm->d_hacc, -1.0, gm->w,
                    gm->w, n, gm->d_norm_partial);
          }
        }
        PLAUNCH(ctx, B200_KID_GIVENS, 0.0, givens_kernel, 1, GM_THREADS, 0, gm->d_state, k, G, norm_partial, gm->d_h, gm->d_R, gm->d_cs, gm->d_sn, gm->d_z,
                gm_hraw(gm, k));
        PLAUNCH(ctx, B200_KID_NORMALIZE, 2.0 * Bv, normalize_kernel, ew_grid, GM_THREADS, 0, gm->d_state, 1, gm->w, gm->V[k], n);
      }
      CHECK_LAUNCH(ctx);
      const bool must_check = (k % check_every == 0) || (iters_total + k >= itmax) || (restart_len > 0 && k >= restart_len);
      if (must_check) {
        B200_TRY(gm_fetch_state(gm));
        if (gm->h_state->status != 0) { cycle_status = gm->h_state->status; k = gm->h_state->k; break; }
      }
    }
    if (oom) {
      B200_TRY(gm_fetch_state(gm));
      if (gm->h_state->status != 0) { cycle_status = gm->h_state->status; k = gm->h_state->k; }
      else if (k >= 16) { cycle_status = -1; }  // implicit restart with the basis that fits
      else { cycle_status = B200_LS_OUT_OF_MEMORY; }
      oom = 0;
    }
    nmatvec += k;
    iters_total += k;
    // algorithmic bytes of this cycle (DESIGN.md §kernels): per Arnoldi step j: operator 3 Bv, normalise 2 Bv and
    //   CGS (2j+2) Bv | CGS2 (4j+4) Bv | MGS (3j+1) Bv (dot pass reads v_{i+1}, update pass reads v_i, w read+written)
    for (int j = 1; j <= k; ++j) {
      double orthb = (orth == B200_ORTH_CGS) ? (2.0 * j + 2.0) : (orth == B200_ORTH_CGS2) ? (4.0 * j + 4.0) : (3.0 * j + 1.0);
      if (resident) bytes += resident_step_bytes(rs.base.passes, j, Bv);
      else bytes += (3.0 + 2.0 + orthb) * Bv;
    }
    // x += V_k y
    if (k > 0 && cycle_status != B200_LS_NONFINITE) {
      LAUNCH(ctx, backsolve_kernel, 1, GM_THREADS, sizeof(double) * (k + 1), gm->d_state, gm->d_R, gm->d_z, gm->d_y, gm->kcap);
      if (Pr) {  // x += N^-1 (V_k y)
        CUDA_TRY(ctx, cudaMemsetAsync(gm->pt1, 0, sizeof(double) * n, ctx->stream));
        PLAUNCH(ctx, B200_KID_UPDATE, (k + 2.0) * Bv, update_kernel, G, GM_THREADS, sizeof(double) * (k + 32), gm->d_state, 1, (const double* const*)gm->d_Vptrs, k, gm->d_y, 1.0,
               gm->pt1, gm->pt1, n, (double*)nullptr);
        B200_TRY(b200i_linop_apply(Pr, gm->pt1, gm->pt2));
        B200_TRY(b200_axpy(ctx, n, 1.0, gm->pt2, x));
        bytes += 6 * Bv;
      } else {
      PLAUNCH(ctx, B200_KID_UPDATE, (k + 2.0) * Bv, update_kernel, G, GM_THREADS, sizeof(double) * (k + 32), gm->d_state, 1, (const double* const*)gm->d_Vptrs, k, gm->d_y, 1.0,
             x, x, n, (double*)nullptr);
      }
      CHECK_LAUNCH(ctx);
      bytes += (k + 2.0) * Bv;
      have_x = true;
    }
    if (cycle_status == -1) {  // restart: next cycle starts from the current x
      ++restarts;
      GmresState* hs = gm->h_state;
      hs->iter_base = (int32_t)iters_total;
      hs->status = 0;
      hs->k = 0;
      CUDA_TRY(ctx, cudaMemcpyAsync(gm->d_state, hs, sizeof(GmresState), cudaMemcpyHostToDevice, ctx->stream));
      CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
      continue;
    }
    final_status = cycle_status;
    break;
  }
  B200_TRY(gm_fetch_state(gm));
  if (resident && final_status == B200_LS_NONFINITE) {  // tell an exchange time-out (bounded spin) from a numerical NaN / Inf
    int flag = 0;
    CUDA_TRY(ctx, cudaMemcpy(&flag, gm->d_err, sizeof(int), cudaMemcpyDeviceToHost));
    if (flag) ctx->fail(B200_OK, "resident GMRES engine: a cross-CTA exchange timed out (bounded spin); the solve is reported as B200_LS_NONFINITE", __FILE__, __LINE__);
  }
  st_local.status = final_status;
  st_local.iters = (int32_t)iters_total;
  st_local.nmatvec = nmatvec;
  st_local.restarts = restarts;
  st_local.rnorm0 = gm->h_state->rnorm0;
  st_local.rnorm = gm->h_state->rnorm;
  st_local.tol = gm->h_state->tol;
  st_local.bytes = bytes;
  if (stats) *stats = st_local;
  return B200_OK;
}
}  // extern "C"
