// ens_batched.cu — batched Newton-GMRES for the ensemble path (SURVEY.md §8a row a11, §8e; BASELINE config 5):
// one CTA per trajectory, persistent over a work queue, the WHOLE NewtonRaphson solve of a trajectory inside one kernel.
//
// Semantics per trajectory = the single-system driver of newton.cu (NewtonRaphson, matrix-free exact JVP, GMRES with
// tolerances inherited from the nonlinear solve, AbsNormSafeBest termination, optional Eisenstat-Walker forcing), i.e.
// what `solve(ensembleprob, NewtonRaphson(linsolve = KrylovJL_GMRES()), EnsembleThreads(); trajectories)` does per
// trajectory in the reference (test/PolyAlgorithms/core_tests__item6.jl:3-20).
//
// Option sets batched here (b200i_ens_batched_supported): exact JVP; unrestarted GMRES with MGS or CGS2 (MGS applied twice),
// any itmax / atol / rtol, optional EW forcing; termination AbsNorm, AbsNormSafe or AbsNormSafeBest on the inf-norm with the
// default step-stall window (32); no maxtime; N <= 32.  Every other option set (the Norm / Rel / Abs modes, the L2 norm,
// another stall window, one-pass CGS, a wall-clock limit, FD-JVP, warm start, restart, N > 32) runs each trajectory
// through the general driver of newton.cu instead (b200_ens_solve).  tests/test_gpu_ensemble.py checks both routes.
//
// Design: a 2D N=32 trajectory has n = 2048 unknowns = 16 KB per vector, so a CTA owns a whole trajectory:
//   * iterate u and the current Krylov direction v_k live in shared memory (stencil neighbourhoods are read from there),
//     the vector being orthogonalised w, the residual and the GMRES solution live in registers (8 rows per thread);
//   * the Krylov basis streams through a per-CTA slab in HBM exactly ONCE per Gram-Schmidt pass: because the CTA owns all
//     rows, Gram-Schmidt is done vector by vector (dot -> block reduction -> update while v_i is still in registers),
//     i.e. modified Gram-Schmidt (Krylov.jl's scheme), applied twice when reorthogonalisation is requested; loads of
//     v_{i+1} are issued before the reduction of v_i (register double buffering) so the stream never drains;
//   * Givens recurrence, stopping tests, back substitution, Newton update, residual, termination: all in the CTA;
//     no host round trip, no grid-wide synchronisation, no lock step between trajectories (converged CTAs fetch the
//     next trajectory from an atomic work queue).
// Algorithmic HBM bytes per Arnoldi step j: passes * j * Bv (basis) + Bv (store v_{j+1}) + j * 8 (R column), Bv = 8 n.
#include "common.cuh"
#include <algorithm>
#include <cstdlib>
#include <math.h>

namespace {
constexpr int ENS_LS_BASIS_FULL = 100;  // internal GMRES stop code: the per-CTA basis slab is full (never leaves this file)
constexpr int ET = 256;   // threads per CTA
constexpr int NPT = 8;    // max rows per thread  -> n <= 2048 (N <= 32)

struct EnsParams {
  int N, n, nprob, maxiters, itmax, kcap, passes, term_mode, forcing, ew_safeguard;
  int walk_di, walk_dj;  // ET mod N, ET div N (row walk of the stencil functions)
  double a, abstol, gm_atol, gm_rtol;
  double ew_eta0, ew_eta_max, ew_gamma, ew_alpha, ew_safeguard_threshold;
  int64_t slab;  // doubles per CTA workspace slab
  int npad;
};

struct CtaState {  // shared-memory scalars, written by thread 0, read after a barrier
  double rnorm, tol, inv_h, hbis, beta;
  int gstatus;
};

__device__ __forceinline__ double blk_sum_all(double v, double (*red)[ET / 32], int& phase) {
  // deterministic block sum, result in every thread; one barrier per call (buffers alternate)
  v = warp_sum(v);
  double* buf = red[phase & 1];
  if ((threadIdx.x & 31) == 0) buf[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
#pragma unroll
  for (int q = 0; q < ET / 32; ++q) s += buf[q];
  phase++;
  return s;
}
__device__ __forceinline__ double blk_max_all(double v, double (*red)[ET / 32], int& phase) {
  v = warp_max(v);
  double* buf = red[phase & 1];
  if ((threadIdx.x & 31) == 0) buf[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
#pragma unroll
  for (int q = 0; q < ET / 32; ++q) s = fmax(s, buf[q]);
  phase++;
  return s;
}

__device__ __forceinline__ void sym_givens_e(double a, double b, double& c, double& s, double& rho) {
  if (b == 0.0) { c = (a == 0.0) ? 1.0 : (a > 0 ? 1.0 : -1.0); s = 0.0; rho = fabs(a); }
  else if (a == 0.0) { c = 0.0; s = (b > 0 ? 1.0 : -1.0); rho = fabs(b); }
  else if (fabs(b) > fabs(a)) { const double t = a / b; s = (b > 0 ? 1.0 : -1.0) / sqrt(1.0 + t * t); c = s * t; rho = b / s; }
  else { const double t = b / a; c = (a > 0 ? 1.0 : -1.0) / sqrt(1.0 + t * t); s = c * t; rho = a / c; }
}

// Grid coordinates (i, j) and species s of this thread's rows r = tid + ET q without a division per row: one division for q = 0, then
// the walk r += ET advances (i, j) by (ET mod N, ET div N) with carries; j wrapping past N is the species boundary (r >= N^2).
#define ENS_ROW_WALK_BEGIN(P, N, NC)                                                      \
  int rw_s = (int)threadIdx.x >= (NC), rw_j, rw_i;                                         \
  {                                                                                        \
    const int c_ = (int)threadIdx.x - rw_s * (NC);                                         \
    rw_j = c_ / (N);                                                                       \
    rw_i = c_ - rw_j * (N);                                                                \
    while (rw_j >= (N)) { rw_j -= (N); ++rw_s; }                                           \
  }
#define ENS_ROW_WALK_STEP(q, N)                                                            \
  if ((q) > 0) {                                                                           \
    rw_i += P.walk_di; rw_j += P.walk_dj;                                                  \
    if (rw_i >= (N)) { rw_i -= (N); ++rw_j; }                                              \
    while (rw_j >= (N)) { rw_j -= (N); ++rw_s; }                                           \
  }
// residual rows of this thread from the shared-memory iterate (brusselator_2d_loop, sparsity_tests__item1.jl:13-36)
__device__ __forceinline__ void ens_residual(const EnsParams& P, double A, double B, const double* __restrict__ us,
                                             const double* __restrict__ forcing, double (&f)[NPT]) {
  const int N = P.N, NC = N * N;
  ENS_ROW_WALK_BEGIN(P, N, NC)
#pragma unroll
  for (int q = 0; q < NPT; ++q) {
    const int r = threadIdx.x + ET * q;
    f[q] = 0.0;
    ENS_ROW_WALK_STEP(q, N)
    if (r < P.n) {
      const int s = rw_s, c = r - s * NC;
      const int i = rw_i, j = rw_j;
      const int ip = (i + 1 == N) ? 0 : i + 1, im = (i == 0) ? N - 1 : i - 1;
      const int jp = (j + 1 == N) ? 0 : j + 1, jm = (j == 0) ? N - 1 : j - 1;
      const double* x = us + s * NC;
      const double lap = x[im + N * j] + x[ip + N * j] + x[i + N * jp] + x[i + N * jm] - 4.0 * x[c];
      const double uc = us[c], vc = us[c + NC];
      const double uuv = uc * uc * vc;
      f[q] = s ? (P.a * lap + A * uc - uuv) : (P.a * lap + B + uuv - (A + 1.0) * uc + forcing[c]);
    }
  }
}
// exact-tangent JVP rows of this thread: direction d in shared memory, state u in shared memory
__device__ __forceinline__ void ens_jvp(const EnsParams& P, double A, const double* __restrict__ us, const double* __restrict__ ds,
                                        double (&w)[NPT]) {
  const int N = P.N, NC = N * N;
  ENS_ROW_WALK_BEGIN(P, N, NC)
#pragma unroll
  for (int q = 0; q < NPT; ++q) {
    const int r = threadIdx.x + ET * q;
    w[q] = 0.0;
    ENS_ROW_WALK_STEP(q, N)
    if (r < P.n) {
      const int s = rw_s, c = r - s * NC;
      const int i = rw_i, j = rw_j;
      const int ip = (i + 1 == N) ? 0 : i + 1, im = (i == 0) ? N - 1 : i - 1;
      const int jp = (j + 1 == N) ? 0 : j + 1, jm = (j == 0) ? N - 1 : j - 1;
      const double* x = ds + s * NC;
      const double lap = x[im + N * j] + x[ip + N * j] + x[i + N * jp] + x[i + N * jm] - 4.0 * x[c];
      const double uc = us[c], vc = us[c + NC], dc = ds[c], ec = ds[c + NC];
      const double uv2 = 2.0 * uc * vc, uu = uc * uc;
      w[q] = s ? (P.a * lap + (A - uv2) * dc - uu * ec) : (P.a * lap + (uv2 - (A + 1.0)) * dc + uu * ec);
    }
  }
}

__global__ void __launch_bounds__(ET, 2) ens_newton_kernel(EnsParams P, const double* __restrict__ u0, const double* __restrict__ Aarr,
                                                            const double* __restrict__ Barr, const double* __restrict__ forcing,
                                                            double* __restrict__ u_out, double* __restrict__ resid_inf,
                                                            int32_t* __restrict__ retcodes, int32_t* __restrict__ nsteps_out,
                                                            int32_t* __restrict__ njvp_out, double* __restrict__ ws, int* __restrict__ counter) {
  extern __shared__ double sm[];
  double* us = sm;                    // iterate u            [npad]
  double* vk = us + P.npad;           // current direction    [npad]
  double* hcol = vk + P.npad;         // Hessenberg column    [kcap + 2]
  double* cs = hcol + P.kcap + 2;     // Givens               [kcap + 2]
  double* sn = cs + P.kcap + 2;
  double* zs = sn + P.kcap + 2;       // rotated rhs          [kcap + 2]
  double* obj_trace = zs + P.kcap + 2;  // [100]
  double* step_trace = obj_trace + 100; // [32]
  double(*red)[ET / 32] = reinterpret_cast<double(*)[ET / 32]>(step_trace + 32);  // [2][8]
  __shared__ CtaState st;
  __shared__ int cur_problem;
  int phase = 0;
  const int n = P.n;
  double* slab = ws + (int64_t)blockIdx.x * P.slab;
  double* Vg = slab;                                   // (kcap + 1) vectors of npad doubles
  double* Rg = slab + (int64_t)(P.kcap + 1) * P.npad;  // packed upper triangular, column k (1-based) at (k-1)k/2

  for (;;) {
    if (threadIdx.x == 0) cur_problem = atomicAdd(counter, 1);
    __syncthreads();
    const int m = cur_problem;
    __syncthreads();
    if (m >= P.nprob) break;
    const double A = Aarr[m], B = Barr[m];
    const double* u0m = u0 + (int64_t)m * n;
    double* uom = u_out + (int64_t)m * n;
    // ---- __init (solve.jl:191-284): u = u0, fu = f(u) (nf not bumped), best = ||fu||_inf, best_u = u
    for (int r = threadIdx.x; r < n; r += ET) { const double v = u0m[r]; us[r] = v; uom[r] = v; }
    __syncthreads();
    double f[NPT];
    ens_residual(P, A, B, us, forcing, f);
    double fmx = 0.0;
#pragma unroll
    for (int q = 0; q < NPT; ++q) fmx = fmax(fmx, abs_nf(f[q]));
    double objective = blk_max_all(fmx, red, phase);
    double best = objective;
    int retcode = B200_RC_DEFAULT, nsteps = 0, njvp = 0, tc_nsteps = 0, force_stop = 0;
    bool rolled_back_needed = false;
    double eta = P.ew_eta0, rnorm_nl = 0.0, rnorm_nl_prev = 0.0;
    while (!force_stop && nsteps < P.maxiters) {
      // ================= descent: GMRES on J(u) x = fu, x0 = 0 (newton.jl:97-141) =================
      double gm_rtol = P.gm_rtol;
      double fsq = 0.0;
#pragma unroll
      for (int q = 0; q < NPT; ++q) fsq = fma(f[q], f[q], fsq);
      const double beta = sqrt(blk_sum_all(fsq, red, phase));
      if (P.forcing) {  // eisenstat_walker.jl:42-87 (internalnorm = L2)
        if (nsteps == 0) { eta = P.ew_eta0; rnorm_nl = rnorm_nl_prev = beta; }
        else {
          const double eta_prev = eta;
          eta = P.ew_gamma * pow(rnorm_nl / rnorm_nl_prev, P.ew_alpha);
          if (P.ew_safeguard) { const double sg = P.ew_gamma * pow(eta_prev, P.ew_alpha); if (sg > P.ew_safeguard_threshold && sg > eta) eta = sg; }
          eta = fmin(fmax(eta, 0.0), P.ew_eta_max);
        }
        gm_rtol = eta;
        rnorm_nl_prev = rnorm_nl;  // post_step_forcing!: fu is still the residual at the pre-update iterate
        rnorm_nl = beta;
      }
      const double tol = P.gm_atol + gm_rtol * beta;
      int gstatus = 0, k = 0;
      if (!(beta == beta) || isinf(beta)) gstatus = B200_LS_NONFINITE;
      else if (beta <= tol) gstatus = B200_LS_SOLVED;
      if (gstatus == 0) {
        const double binv = 1.0 / beta;
#pragma unroll
        for (int q = 0; q < NPT; ++q) {
          const int r = threadIdx.x + ET * q;
          if (r < n) { const double v = f[q] * binv; vk[r] = v; Vg[r] = v; }
        }
        if (threadIdx.x == 0) zs[0] = beta;
        __syncthreads();
      }
      while (gstatus == 0) {
        ++k;
        double w[NPT];
        ens_jvp(P, A, us, vk, w);
        ++njvp;
        // ---- (iterated) modified Gram-Schmidt, one basis read per pass
        for (int pass = 0; pass < P.passes; ++pass) {
          double vn[NPT], vc[NPT];
#pragma unroll
          for (int q = 0; q < NPT; ++q) { const int r = threadIdx.x + ET * q; vn[q] = (r < n) ? Vg[r] : 0.0; }
          for (int i = 0; i < k; ++i) {
#pragma unroll
            for (int q = 0; q < NPT; ++q) vc[q] = vn[q];
            if (i + 1 < k) {
              const double* vnext = Vg + (int64_t)(i + 1) * P.npad;
#pragma unroll
              for (int q = 0; q < NPT; ++q) { const int r = threadIdx.x + ET * q; vn[q] = (r < n) ? vnext[r] : 0.0; }
            }
            double d = 0.0;
#pragma unroll
            for (int q = 0; q < NPT; ++q) d = fma(vc[q], w[q], d);
            const double h = blk_sum_all(d, red, phase);
#pragma unroll
            for (int q = 0; q < NPT; ++q) w[q] = fma(-h, vc[q], w[q]);
            if (threadIdx.x == 0) hcol[i] = (pass == 0) ? h : hcol[i] + h;
          }
        }
        double wsq = 0.0;
#pragma unroll
        for (int q = 0; q < NPT; ++q) wsq = fma(w[q], w[q], wsq);
        const double hbis = sqrt(blk_sum_all(wsq, red, phase));
        // ---- Givens recurrence on the new column (thread 0), Krylov.jl reflection convention
        if (threadIdx.x == 0) {
          for (int i = 0; i + 1 < k; ++i) {
            const double rt = cs[i] * hcol[i] + sn[i] * hcol[i + 1];
            hcol[i + 1] = sn[i] * hcol[i] - cs[i] * hcol[i + 1];
            hcol[i] = rt;
          }
          double c, s_, rho;
          sym_givens_e(hcol[k - 1], hbis, c, s_, rho);
          cs[k - 1] = c; sn[k - 1] = s_; hcol[k - 1] = rho;
          const double zeta = s_ * zs[k - 1];
          zs[k - 1] = c * zs[k - 1];
          zs[k] = zeta;
          const double rn = fabs(zeta);
          int gs = 0;
          if (!(rn == rn) || isinf(rn) || !(hbis == hbis) || isinf(hbis)) gs = B200_LS_NONFINITE;
          else if (rn <= tol) gs = B200_LS_SOLVED;
          else if (k >= P.itmax) gs = B200_LS_MAXITERS;
          else if (k >= P.kcap) gs = ENS_LS_BASIS_FULL;  // basis slab exhausted before itmax: hand the trajectory to the general driver
          else if (hbis <= 1.8189894035458565e-12) gs = B200_LS_BREAKDOWN;
          st.gstatus = gs; st.rnorm = rn; st.inv_h = hbis > 0.0 ? 1.0 / hbis : 0.0;
        }
        __syncthreads();
        gstatus = st.gstatus;
        double* Rk = Rg + (int64_t)(k - 1) * k / 2;
        for (int i = threadIdx.x; i < k; i += ET) Rk[i] = hcol[i];
        if (gstatus == 0) {
          const double inv = st.inv_h;
          double* vnew = Vg + (int64_t)k * P.npad;
#pragma unroll
          for (int q = 0; q < NPT; ++q) {
            const int r = threadIdx.x + ET * q;
            if (r < n) { const double v = w[q] * inv; vk[r] = v; vnew[r] = v; }
          }
        }
        __syncthreads();
      }
      if (gstatus == ENS_LS_BASIS_FULL) { retcode = B200I_ENS_RC_DEFERRED; force_stop = 1; break; }
      if (gstatus == B200_LS_NONFINITE) {  // linear solve failed with a current Jacobian (solve.jl:367-372)
        retcode = B200_RC_INTERNAL_LINSOLVE_FAILED;
        force_stop = 1;
        ++nsteps;
        break;
      }
      // ---- y = R^{-1} z (column-oriented back substitution), x = V_k y
      __syncthreads();
      for (int i = k - 1; i >= 0; --i) {
        const double* Ri = Rg + (int64_t)i * (i + 1) / 2;
        const double d = Ri[i];
        const double yi = (d == 0.0) ? 0.0 : zs[i] / d;
        __syncthreads();
        if (threadIdx.x == 0) zs[i] = yi;
        for (int j = threadIdx.x; j < i; j += ET) zs[j] -= Ri[j] * yi;
        __syncthreads();
      }
      double x[NPT];
#pragma unroll
      for (int q = 0; q < NPT; ++q) x[q] = 0.0;
      for (int i = 0; i < k; ++i) {
        const double yi = zs[i];
        const double* vi = Vg + (int64_t)i * P.npad;
#pragma unroll
        for (int q = 0; q < NPT; ++q) { const int r = threadIdx.x + ET * q; if (r < n) x[q] = fma(yi, vi[r], x[q]); }
      }
      // ================= u += du, du = -x ; fu = f(u) ; termination (solve.jl:436-452) =================
      double dsq = 0.0;
      __syncthreads();
#pragma unroll
      for (int q = 0; q < NPT; ++q) {
        const int r = threadIdx.x + ET * q;
        if (r < n) { us[r] -= x[q]; dsq = fma(x[q], x[q], dsq); }
      }
      __syncthreads();
      ens_residual(P, A, B, us, forcing, f);
      fmx = 0.0;
#pragma unroll
      for (int q = 0; q < NPT; ++q) fmx = fmax(fmx, abs_nf(f[q]));
      objective = blk_max_all(fmx, red, phase);
      const double du_norm = sqrt(blk_sum_all(dsq, red, phase));
      ++nsteps;
      // AbsNorm* termination (termination_conditions.jl:243-336), evaluated redundantly and identically by every thread
      if (P.term_mode == B200_TERM_ABS_NORM) {
        if (objective <= P.abstol) { retcode = B200_RC_SUCCESS; force_stop = 1; }
      } else if (!isfinite(objective)) {
        retcode = B200_RC_UNSTABLE; force_stop = 1;
      } else {
        if (P.term_mode == B200_TERM_ABS_NORM_SAFE_BEST && objective < best) {
          best = objective;
          for (int r = threadIdx.x; r < n; r += ET) uom[r] = us[r];
          rolled_back_needed = false;
        } else if (P.term_mode == B200_TERM_ABS_NORM_SAFE_BEST) {
          rolled_back_needed = true;
        }
        if (objective <= P.abstol) { retcode = B200_RC_SUCCESS; force_stop = 1; }
        else {
          tc_nsteps += 1;
          if (threadIdx.x == 0) { obj_trace[(tc_nsteps - 1) % 100] = objective; step_trace[(tc_nsteps - 1) % 32] = du_norm; }
          __syncthreads();
          if (objective <= 3.0 * P.abstol && tc_nsteps > 100) {
            double mn = INFINITY, mx = -INFINITY;
            for (int i = 0; i < 100; ++i) { mn = fmin(mn, obj_trace[i]); mx = fmax(mx, obj_trace[i]); }
            if (mn < 1.3 * mx) { retcode = B200_RC_STALLED; force_stop = 1; }
          }
          if (!force_stop && tc_nsteps > 32) {
            double mx = 0.0;
            for (int i = 0; i < 32; ++i) mx = fmax(mx, step_trace[i]);
            if (mx <= P.abstol) { retcode = B200_RC_STALLED; force_stop = 1; }
          }
        }
      }
    }
    if (retcode == B200_RC_DEFAULT) retcode = (nsteps >= P.maxiters) ? B200_RC_MAXITERS : B200_RC_SUCCESS;
    // ---- update_from_termination_cache! (termination_conditions.jl:440-453): Best modes return the best iterate
    if (P.term_mode == B200_TERM_ABS_NORM_SAFE_BEST) {
      if (rolled_back_needed) {  // the last iterate is not the best one: recompute the residual at the stored best u
        __syncthreads();
        for (int r = threadIdx.x; r < n; r += ET) us[r] = uom[r];
        __syncthreads();
        ens_residual(P, A, B, us, forcing, f);
        fmx = 0.0;
#pragma unroll
        for (int q = 0; q < NPT; ++q) fmx = fmax(fmx, abs_nf(f[q]));
        objective = blk_max_all(fmx, red, phase);
      }
    } else {
      for (int r = threadIdx.x; r < n; r += ET) uom[r] = us[r];
    }
    if (threadIdx.x == 0) {
      if (retcode == B200I_ENS_RC_DEFERRED) atomicAdd(counter + 1, 1);
      resid_inf[m] = objective;
      retcodes[m] = retcode;
      nsteps_out[m] = nsteps;
      njvp_out[m] = njvp;
    }
    __syncthreads();
  }
}

size_t ens_smem_bytes(const EnsParams& P) {
  return sizeof(double) * ((size_t)2 * P.npad + 4 * (size_t)(P.kcap + 2) + 100 + 32 + 2 * (ET / 32));
}
}  // namespace

// The option sets the kernel implements exactly; everything else goes to the general driver (b200_ens_solve's sequential route).
// Termination: the three AbsNorm modes on the inf-norm, with the Safe modes' step-stall window at its default of 32 (the
// window is fixed in the kernel; a non-Safe mode has none, so its setting does not matter).  No wall-clock limit.
int32_t b200i_ens_batched_supported(int32_t N, const b200_newton_opts* o) {
  if (2 * N * N > ET * NPT) return 0;
  if (o->jvp_mode != B200_JVP_EXACT || o->gmres.warm_start || o->gmres.restart > 0) return 0;
  if (o->gmres.orth != B200_ORTH_MGS && o->gmres.orth != B200_ORTH_CGS2) return 0;
  const int t = o->termination;
  if (t != B200_TERM_ABS_NORM && t != B200_TERM_ABS_NORM_SAFE && t != B200_TERM_ABS_NORM_SAFE_BEST) return 0;
  if (o->term_norm != B200_NORM_INF) return 0;
  if (t != B200_TERM_ABS_NORM && o->term_max_stalled_steps != 0 && o->term_max_stalled_steps != 32) return 0;
  if (o->maxtime > 0.0) return 0;
  return 1;
}

int32_t b200i_ens_batched_solve(b200_ctx* ctx, int32_t N, int32_t nprob, double alpha, const b200_newton_opts* o, const double* u0,
                                const double* A, const double* B, double* u_out, double* resid_inf, int32_t* retcodes, int32_t* nsteps,
                                int32_t* njvp, void** workspace, size_t* workspace_bytes, int32_t* n_deferred) {
  EnsParams P;
  memset(&P, 0, sizeof(P));
  P.N = N; P.n = 2 * N * N; P.nprob = nprob;
  P.walk_di = ET % N; P.walk_dj = ET / N;
  P.npad = (P.n + 1) & ~1;
  P.maxiters = o->maxiters > 0 ? o->maxiters : 1000;
  P.abstol = o->abstol > 0 ? o->abstol : 3.0e-13;
  const double reltol = o->reltol > 0 ? o->reltol : 3.0e-13;
  P.gm_atol = o->gmres.atol > 0 ? o->gmres.atol : P.abstol;
  P.gm_rtol = o->gmres.rtol > 0 ? o->gmres.rtol : reltol;
  P.itmax = o->gmres.itmax > 0 ? o->gmres.itmax : P.n;
  // per-CTA basis slab: 512 columns unless B200_ENS_BASIS_COLUMNS says otherwise (memory knob: the slab is (kcap + 1) n doubles per
  // resident CTA).  A trajectory that needs more columns than this is not truncated: it is redone by the general driver.
  int slab_cols = 512;
  if (const char* e = getenv("B200_ENS_BASIS_COLUMNS")) { const int v = atoi(e); if (v >= 2) slab_cols = v; }
  P.kcap = std::min(std::min(P.n, P.itmax), slab_cols);
  P.passes = (o->gmres.orth == B200_ORTH_MGS) ? 1 : 2;  // MGS, or MGS applied twice (reorthogonalisation) for CGS2
  P.term_mode = o->termination;
  P.forcing = o->forcing == B200_FORCING_EW2;
  P.ew_eta0 = o->ew_eta0; P.ew_eta_max = o->ew_eta_max; P.ew_gamma = o->ew_gamma; P.ew_alpha = o->ew_alpha;
  P.ew_safeguard = o->ew_safeguard; P.ew_safeguard_threshold = o->ew_safeguard_threshold;
  const double dx = 1.0 / (double)(N - 1);
  P.a = alpha / (dx * dx);
  P.slab = (int64_t)(P.kcap + 1) * P.npad + (int64_t)P.kcap * (P.kcap + 1) / 2 + 16;
  const size_t smem = ens_smem_bytes(P);
  CUDA_TRY(ctx, cudaFuncSetAttribute(ens_newton_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  CUDA_TRY(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ens_newton_kernel, ET, smem));
  if (per_sm < 1) return ctx->fail(B200_ERR_UNSUPPORTED, "ensemble kernel does not fit on an SM", __FILE__, __LINE__);
  const int grid = std::min(nprob, per_sm * ctx->sm_count);
  // workspace: per-CTA slabs + the forcing plane + the work-queue counter
  const size_t need = sizeof(double) * ((size_t)grid * P.slab + (size_t)N * N) + 64;
  if (*workspace_bytes < need) {
    if (*workspace) { CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream)); cudaFree(*workspace); *workspace = nullptr; *workspace_bytes = 0; }
    if (cudaMalloc(workspace, need) != cudaSuccess) { cudaGetLastError(); return ctx->fail(B200_ERR_NOMEM, "ensemble workspace allocation failed", __FILE__, __LINE__); }
    *workspace_bytes = need;
  }
  double* ws = reinterpret_cast<double*>(*workspace);
  double* d_forcing = ws + (size_t)grid * P.slab;
  int* d_counter = reinterpret_cast<int*>(d_forcing + (size_t)N * N);
  std::vector<double> forcing((size_t)N * N);
  const double r2 = 0.1 * 0.1;
  for (int j = 0; j < N; ++j)
    for (int i = 0; i < N; ++i) {
      volatile double x = (double)i / (double)(N - 1), y = (double)j / (double)(N - 1);
      volatile double dx2 = (x - 0.3) * (x - 0.3), dy2 = (y - 0.6) * (y - 0.6);
      volatile double s = dx2 + dy2;
      forcing[(size_t)i + (size_t)N * j] = (s <= r2) ? 5.0 : 0.0;
    }
  CUDA_TRY(ctx, cudaMemcpyAsync(d_forcing, forcing.data(), sizeof(double) * forcing.size(), cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(ctx, cudaMemsetAsync(d_counter, 0, 2 * sizeof(int), ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));  // `forcing` is a host temporary
  PLAUNCH(ctx, B200_KID_RESIDENT, 0.0, ens_newton_kernel, grid, ET, smem, P, u0, A, B, (const double*)d_forcing, u_out, resid_inf, retcodes, nsteps,
          njvp, ws, d_counter);
  CHECK_LAUNCH(ctx);
  // trajectories whose Krylov basis outgrew the per-CTA slab (kcap < min(itmax, n)) come back marked B200I_ENS_RC_DEFERRED
  int hits = 0;
  CUDA_TRY(ctx, cudaMemcpyAsync(&hits, d_counter + 1, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  *n_deferred = hits;
  return B200_OK;
}
