// problems.cu — residual f(u), exact-tangent JVP J(u)v, VJP J(u)'w and the fused finite-difference JVP for the
// built-in problems (SURVEY.md §8a rows a1, a2; kernels K1, K2).
//
//   2D/3D Brusselator  : lib/NonlinearSolveFirstOrder/test/sparsity_tests__item1.jl:7-50 (3D extension: SURVEY.md §A.2)
//   quadratic u.^2 .- p: common/common_rootfind_testing.jl:15
//   tridiagonal quad.  : lib/NonlinearSolveFirstOrder/test/rootfind_tests__item20.jl:6-29
//   callback           : NonlinearFunction{true}(f!; jvp = jvp!)  (SciMLJacobianOperators.jl:366-431 takes f.jvp verbatim)
//
// Layout: species-planar, i fastest: idx(i,j[,k],s) = i + N j [+ N^2 k] + N^dim s  (Julia column-major (N,N[,N],2)).
// The JVP is the exact tangent of the residual expression (what DI.pushforward! with ForwardDiff computes,
// SciMLJacobianOperators.jl:396-414), not a finite difference; b200_jvp_fd is the AutoFiniteDiff analogue.
#include "common.cuh"
#include <math.h>
#include <float.h>
#include <algorithm>

namespace {
constexpr int PB_THREADS = 256;

enum { M_RESID = 1, M_JVP = 2, M_VJP = 4, M_NORM = 8, M_FD = 16 };

struct BrussParams {
  int N;
  double a, A, B;
};

// Point formulas shared by every Brusselator kernel of this file.  Written with explicit round-to-nearest intrinsics so that the
// compiler's FMA contraction cannot differ from kernel to kernel: the fused residual+JVP kernel, the halo-tile kernels and the
// 2D kernel (a z-independent 3D state) then agree bit for bit, which tests/test_gpu_fullsize.py asserts.
__device__ __forceinline__ void bruss_react(double uc, double vc, double A, double& j00, double& j01, double& j10, double& j11) {
  const double uv2 = __dmul_rn(__dmul_rn(2.0, uc), vc), uu = __dmul_rn(uc, uc);
  j00 = __dadd_rn(uv2, -(A + 1.0));
  j01 = uu;
  j10 = __dadd_rn(A, -uv2);
  j11 = -uu;
}
__device__ __forceinline__ double lap_plane(double im, double ip, double jp, double jm, double c) {
  return __fma_rn(-4.0, c, __dadd_rn(__dadd_rn(__dadd_rn(im, ip), jp), jm));
}
__device__ __forceinline__ double lap_z(double kp, double km, double c) { return __fma_rn(-2.0, c, __dadd_rn(kp, km)); }  // exactly 0 for a z-independent state
__device__ __forceinline__ void bruss_resid(const BrussParams& P, double lapu, double lapv, double uc, double vc, double fo, double& f0, double& f1) {
  const double uuv = __dmul_rn(__dmul_rn(uc, uc), vc);
  f0 = __dadd_rn(__fma_rn(-(P.A + 1.0), uc, __dadd_rn(__fma_rn(P.a, lapu, P.B), uuv)), fo);
  f1 = __dadd_rn(__fma_rn(P.a, lapv, __dmul_rn(P.A, uc)), -uuv);
}
// (J v) at a cell from the Laplacians of the direction and the 2x2 reaction block; TRANSPOSE: J' w
template <bool TRANSPOSE>
__device__ __forceinline__ void bruss_tangent(const BrussParams& P, double lapd, double lape, double uc, double vc, double dc, double ec, double& o0, double& o1) {
  double j00, j01, j10, j11;
  bruss_react(uc, vc, P.A, j00, j01, j10, j11);
  o0 = __fma_rn(TRANSPOSE ? j10 : j01, ec, __fma_rn(j00, dc, __dmul_rn(P.a, lapd)));
  o1 = __fma_rn(j11, ec, __fma_rn(TRANSPOSE ? j01 : j10, dc, __dmul_rn(P.a, lape)));
}

// ---- 2D: one thread per cell.  n is small for every 2D configuration (N<=128 -> 256 KB), so the whole state is
// L2/L1 resident and a halo tile buys nothing; the 3D kernel below is the bandwidth-critical one.
template <int MODE>
__global__ void __launch_bounds__(PB_THREADS) bruss2d_kernel(BrussParams P, const double* __restrict__ u, const double* __restrict__ d,
                                                              const double* __restrict__ forcing, double* __restrict__ du,
                                                              double* __restrict__ Jd, double* __restrict__ norm_out,
                                                              const double* __restrict__ eps_ptr) {
  __shared__ double red[32];
  const int N = P.N;
  const int NC = N * N;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  double nrm = 0.0;
  if (c < NC) {
    const int i = c % N, j = c / N;
    const int ip = (i + 1 == N) ? 0 : i + 1, im = (i == 0) ? N - 1 : i - 1;
    const int jp = (j + 1 == N) ? 0 : j + 1, jm = (j == 0) ? N - 1 : j - 1;
    const int cim = im + N * j, cip = ip + N * j, cjp = i + N * jp, cjm = i + N * jm;
    const double uc = u[c], vc = u[c + NC];
    if (MODE & M_RESID) {
      const double lapu = lap_plane(u[cim], u[cip], u[cjp], u[cjm], uc);
      const double lapv = lap_plane(u[cim + NC], u[cip + NC], u[cjp + NC], u[cjm + NC], vc);
      double f0, f1;
      bruss_resid(P, lapu, lapv, uc, vc, forcing[c], f0, f1);
      du[c] = f0;
      du[c + NC] = f1;
      if (MODE & M_NORM) nrm = fmax(abs_nf(f0), abs_nf(f1));
    }
    if (MODE & (M_JVP | M_VJP)) {
      const double dc = d[c], ec = d[c + NC];
      const double lapd = lap_plane(d[cim], d[cip], d[cjp], d[cjm], dc);
      const double lape = lap_plane(d[cim + NC], d[cip + NC], d[cjp + NC], d[cjm + NC], ec);
      double o0, o1;
      bruss_tangent<(MODE & M_VJP) != 0>(P, lapd, lape, uc, vc, dc, ec, o0, o1);
      Jd[c] = o0;
      Jd[c + NC] = o1;
    }
    if (MODE & M_FD) {  // (f(u + eps d) - f(u)) / eps evaluated in one pass over the shared neighbourhood
      const double eps = *eps_ptr;
      const double dc = d[c], ec = d[c + NC];
      const double lapu = u[cim] + u[cip] + u[cjp] + u[cjm] - 4.0 * uc;
      const double lapv = u[cim + NC] + u[cip + NC] + u[cjp + NC] + u[cjm + NC] - 4.0 * vc;
      const double up = uc + eps * dc, vp = vc + eps * ec;
      const double lapup = (u[cim] + eps * d[cim]) + (u[cip] + eps * d[cip]) + (u[cjp] + eps * d[cjp]) + (u[cjm] + eps * d[cjm]) - 4.0 * up;
      const double lapvp = (u[cim + NC] + eps * d[cim + NC]) + (u[cip + NC] + eps * d[cip + NC]) + (u[cjp + NC] + eps * d[cjp + NC]) +
                           (u[cjm + NC] + eps * d[cjm + NC]) - 4.0 * vp;
      const double fo = forcing[c];
      const double f0 = P.a * lapu + P.B + uc * uc * vc - (P.A + 1.0) * uc + fo;
      const double f1 = P.a * lapv + P.A * uc - uc * uc * vc;
      const double g0 = P.a * lapup + P.B + up * up * vp - (P.A + 1.0) * up + fo;
      const double g1 = P.a * lapvp + P.A * up - up * up * vp;
      Jd[c] = (g0 - f0) / eps;
      Jd[c + NC] = (g1 - f1) / eps;
    }
  }
  if (MODE & M_NORM) {
    nrm = block_max(nrm, red);
    if (threadIdx.x == 0) atomic_max_nonneg(norm_out, nrm);
  }
}

// ---- 3D: thread per cell, i fastest -> the centre loads/stores of a warp are one contiguous 256-byte segment per
// species; i+-1 neighbours hit the same lines in L1, j+-1 / k+-1 neighbours are re-reads served by L1/L2 (the whole
// 32 MB state of the N=100 case sits in the 50 MB L2), so HBM traffic stays at the algorithmic 2/3/4 Bv.
template <int MODE>
__global__ void __launch_bounds__(PB_THREADS) bruss3d_kernel(BrussParams P, const double* __restrict__ u, const double* __restrict__ d,
                                                              const double* __restrict__ forcing, double* __restrict__ du,
                                                              double* __restrict__ Jd, double* __restrict__ norm_out,
                                                              const double* __restrict__ eps_ptr) {
  __shared__ double red[32];
  const int N = P.N;
  const int N2 = N * N;
  const int64_t NC = (int64_t)N2 * N;
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  double nrm = 0.0;
  if (c < NC) {
    const int k = (int)(c / N2);
    const int r = (int)(c - (int64_t)k * N2);
    const int j = r / N, i = r - j * N;
    const int64_t cim = c + ((i == 0) ? (N - 1) : -1), cip = c + ((i + 1 == N) ? -(N - 1) : 1);
    const int64_t cjm = c + ((j == 0) ? (int64_t)(N - 1) * N : -N), cjp = c + ((j + 1 == N) ? -(int64_t)(N - 1) * N : N);
    const int64_t ckm = c + ((k == 0) ? (int64_t)(N - 1) * N2 : -N2), ckp = c + ((k + 1 == N) ? -(int64_t)(N - 1) * N2 : N2);
    const double uc = u[c], vc = u[c + NC];
    if (MODE & M_RESID) {
      const double lapu = __dadd_rn(lap_plane(u[cim], u[cip], u[cjp], u[cjm], uc), lap_z(u[ckp], u[ckm], uc));
      const double lapv = __dadd_rn(lap_plane(u[cim + NC], u[cip + NC], u[cjp + NC], u[cjm + NC], vc), lap_z(u[ckp + NC], u[ckm + NC], vc));
      double f0, f1;
      bruss_resid(P, lapu, lapv, uc, vc, forcing[r], f0, f1);
      du[c] = f0;
      du[c + NC] = f1;
      if (MODE & M_NORM) nrm = fmax(abs_nf(f0), abs_nf(f1));
    }
    if (MODE & (M_JVP | M_VJP)) {
      const double dc = d[c], ec = d[c + NC];
      const double lapd = __dadd_rn(lap_plane(d[cim], d[cip], d[cjp], d[cjm], dc), lap_z(d[ckp], d[ckm], dc));
      const double lape = __dadd_rn(lap_plane(d[cim + NC], d[cip + NC], d[cjp + NC], d[cjm + NC], ec), lap_z(d[ckp + NC], d[ckm + NC], ec));
      double o0, o1;
      bruss_tangent<(MODE & M_VJP) != 0>(P, lapd, lape, uc, vc, dc, ec, o0, o1);
      Jd[c] = o0;
      Jd[c + NC] = o1;
    }
    if (MODE & M_FD) {
      const double eps = *eps_ptr;
      const double dc = d[c], ec = d[c + NC];
      const double up = uc + eps * dc, vp = vc + eps * ec;
      const double lapu = (u[cim] + u[cip] + u[cjp] + u[cjm] - 4.0 * uc) + (u[ckp] + u[ckm] - 2.0 * uc);
      const double lapv = (u[cim + NC] + u[cip + NC] + u[cjp + NC] + u[cjm + NC] - 4.0 * vc) + (u[ckp + NC] + u[ckm + NC] - 2.0 * vc);
#define PU(x) (u[x] + eps * d[x])
      const double lapup = (PU(cim) + PU(cip) + PU(cjp) + PU(cjm) - 4.0 * up) + (PU(ckp) + PU(ckm) - 2.0 * up);
      const double lapvp = (PU(cim + NC) + PU(cip + NC) + PU(cjp + NC) + PU(cjm + NC) - 4.0 * vp) + (PU(ckp + NC) + PU(ckm + NC) - 2.0 * vp);
#undef PU
      const double fo = forcing[r];
      const double f0 = P.a * lapu + P.B + uc * uc * vc - (P.A + 1.0) * uc + fo;
      const double f1 = P.a * lapv + P.A * uc - uc * uc * vc;
      const double g0 = P.a * lapup + P.B + up * up * vp - (P.A + 1.0) * up + fo;
      const double g1 = P.a * lapvp + P.A * up - up * up * vp;
      Jd[c] = (g0 - f0) / eps;
      Jd[c + NC] = (g1 - f1) / eps;
    }
  }
  if (MODE & M_NORM) {
    nrm = block_max(nrm, red);
    if (threadIdx.x == 0) atomic_max_nonneg(norm_out, nrm);
  }
}

// ---- 3D, bandwidth-critical form (K1 / K2 of SURVEY.md §8a; north_star: shared-memory halo tile, 16-byte accesses along i,
// fused norm).  At N = 100 a whole kernel moves 32-48 MB — 10-14 us at the H100's HBM peak — so what decides the time is how many
// bytes are in flight from the first microsecond on, not the arithmetic.  Organisation:
//   * a plane (i, j) is N^2 contiguous doubles; the unit of work is a PLANE-CHUNK: TS_L = 2 * TS_THREADS consecutive flat plane
//     positions of one k plane (a thread: two neighbouring cells, one 16-byte access; N even keeps a pair inside one row).
//     The chunks * N plane-chunks are dealt out in contiguous runs to a ONE-WAVE grid (2 CTAs per SM), so every CTA marches
//     over ~N * chunks / grid consecutive k planes of one chunk (two marches when its run crosses a chunk boundary);
//   * a march reads each plane ONCE: planes k-1, k, k+1 of the field whose Laplacian is taken (+ a halo of N positions either
//     side of the chunk, which carries the j -/+ 1 neighbours and both periodic wraps) sit in a shared-memory RING of R plane
//     slots filled by TMA bulk copies.  A dedicated PRODUCER warp issues them (full / empty mbarrier pair per slot); the eight
//     consumer warps never meet at a CTA-wide barrier: each waits for the newest plane, computes, and releases the oldest slot.
//     R - 3 slots are always in flight ahead of the compute, with no registers tied up by loads;
//   * the field that enters through its centre value only (u in the JVP / VJP) rides in the same slot; the forcing plane of
//     the residual is a per-thread constant;
//   * outputs go straight to global memory as 16-byte stores; ||f||_inf is folded into the residual's epilogue.
// HBM traffic: (m + 2) / m of the Laplacian field for a march of m planes (m ~ 7.6 at N = 100 on 264 CTAs: +26 % of ONE of
// the two or three vectors, served from L2 for the most part since neighbouring CTAs read the same planes at the same time).
constexpr int TS_THREADS = 256;
constexpr int TS_L = 2 * TS_THREADS;
constexpr int TS_MAXR = 8;        // ring slots (at most)
constexpr int TS_MAXMARCH = 4;    // marches per CTA (a run crosses at most a few chunk boundaries)

struct TsMarch { int chunk, ka, m, l0; };  // planes ka .. ka + m - 1 of `chunk`; its loads are l0 .. l0 + m + 1 (planes ka - 1 .. ka + m)

template <int MODE>
__global__ void __launch_bounds__(TS_THREADS + 32, 2) bruss3d_ring_kernel(BrussParams P, int R, const double* __restrict__ u, const double* __restrict__ d,
                                                                           const double* __restrict__ forcing, double* __restrict__ out,
                                                                           double* __restrict__ norm_out) {
  extern __shared__ __align__(16) double ts_sm[];
  __shared__ uint64_t full[TS_MAXR], empty[TS_MAXR];   // full: the slot's copies have landed; empty: every consumer thread has read it
  __shared__ TsMarch march[TS_MAXMARCH];
  __shared__ int nmarch_s, nload_s;
  __shared__ double red[32];
  constexpr bool HAS_Y = (MODE & (M_JVP | M_VJP)) != 0;
  const int N = P.N, N2 = N * N, tid = threadIdx.x;
  const int64_t NC = (int64_t)N2 * N;
  const int xrow = TS_L + 2 * N;                       // doubles per species of the Laplacian field in a slot
  const int slot_doubles = 2 * xrow + (HAS_Y ? 2 * TS_L : 0);
  const double* __restrict__ X = (MODE & M_RESID) ? u : d;
  const int chunks = (N2 + TS_L - 1) / TS_L;
  if (tid == TS_THREADS) {
    const int64_t W = (int64_t)chunks * N;
    int64_t w0 = W * blockIdx.x / gridDim.x;
    const int64_t w1 = W * (blockIdx.x + 1) / gridDim.x;
    int nm = 0, l = 0;
    while (w0 < w1 && nm < TS_MAXMARCH) {
      const int c = (int)(w0 / N), ka = (int)(w0 - (int64_t)c * N);
      const int m = (int)min((int64_t)(N - ka), w1 - w0);
      march[nm] = TsMarch{c, ka, m, l};
      l += m + 2;
      w0 += m;
      ++nm;
    }
    nmarch_s = nm; nload_s = l;
    for (int r = 0; r < R; ++r) { mbar_init(&full[r], 1); mbar_init(&empty[r], TS_THREADS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int nmarch = nmarch_s, nload = nload_s;
  double nrm = 0.0;
  if (tid >= TS_THREADS) {
    // ---- producer warp (one lane): load l = plane (ka - 1 + l - l0) of its march's chunk into slot l mod R, as soon as the
    //      consumers have released the slot's previous occupant
    if (tid == TS_THREADS) {
      int slot_i = 0, round = 0, mi = 0;
      for (int l = 0; l < nload; ++l) {
        if (round > 0) mbar_wait(&empty[slot_i], (unsigned)((round - 1) & 1));
        while (mi + 1 < nmarch && l >= march[mi + 1].l0) ++mi;
        const TsMarch mc = march[mi];
        int kk = mc.ka - 1 + (l - mc.l0);
        kk = (kk < 0) ? kk + N : (kk >= N ? kk - N : kk);
        const int p0 = mc.chunk * TS_L;
        double* slot = ts_sm + (size_t)slot_i * slot_doubles;
        uint64_t* bar = &full[slot_i];
        // region [p0 - N, p0 + TS_L + N) of the plane, periodic in the flat plane index: at most one wrap (N2 >= TS_L + 2N)
        int q0 = p0 - N;
        if (q0 < 0) q0 += N2;
        const int first = min(xrow, N2 - q0), second = xrow - first;
        const int ylen = HAS_Y ? min(TS_L, N2 - p0) : 0;
        mbar_expect_tx(bar, (unsigned)(2 * xrow * 8 + 2 * ylen * 8));
#pragma unroll
        for (int s = 0; s < 2; ++s) {
          const double* src = X + s * NC + (int64_t)kk * N2;
          tma_bulk_load(slot + s * xrow, src + q0, (unsigned)(first * 8), bar);
          if (second > 0) tma_bulk_load(slot + s * xrow + first, src, (unsigned)(second * 8), bar);
          if (HAS_Y) tma_bulk_load(slot + 2 * xrow + s * TS_L, u + s * NC + (int64_t)kk * N2 + p0, (unsigned)(ylen * 8), bar);
        }
        if (++slot_i == R) { slot_i = 0; ++round; }
      }
    }
  } else {
    // ---- consumer warps: no CTA-wide barrier in the march — a warp waits for the newest plane, computes, and hands the oldest
    //      slot back to the producer
    for (int mi = 0; mi < nmarch; ++mi) {
      const TsMarch mc = march[mi];
      const int p = mc.chunk * TS_L + 2 * tid;
      const bool valid = p < N2;
      int ileft = -1, iright = 2;  // offsets of the i - 1 / i + 2 neighbours from this thread's pair (periodic in the row)
      double2 fo = {0.0, 0.0};
      if (valid) {
        const int j = p / N, i = p - j * N;
        if (i == 0) ileft = N - 1;
        if (i + 2 == N) iright = 2 - N;
        if (MODE & M_RESID) fo = *reinterpret_cast<const double2*>(forcing + p);
      }
      // ring positions of loads l0, l0 + 1, l0 + 2 (slot, phase parity), advanced incrementally: no division in the march
      int sm_i = mc.l0 % R, pm = (mc.l0 / R) & 1;
      int sc_i = sm_i + 1, pc = pm;
      if (sc_i == R) { sc_i = 0; pc ^= 1; }
      int sp_i = sc_i + 1, pp = pc;
      if (sp_i == R) { sp_i = 0; pp ^= 1; }
      mbar_wait(&full[sm_i], (unsigned)pm);
      mbar_wait(&full[sc_i], (unsigned)pc);
      const double* xoff = ts_sm + N + 2 * tid;
      for (int jj = 0; jj < mc.m; ++jj) {
        const int k = mc.ka + jj;
        mbar_wait(&full[sp_i], (unsigned)pp);
        if (valid) {
          const double* sm_ = xoff + (size_t)sm_i * slot_doubles;
          const double* sc_ = xoff + (size_t)sc_i * slot_doubles;
          const double* sp_ = xoff + (size_t)sp_i * slot_doubles;
          double2 lap[2], xc[2];
#pragma unroll
          for (int s = 0; s < 2; ++s) {
            const double* row = sc_ + s * xrow;  // row[0], row[1]: this thread's cells
            const double2 c2 = *reinterpret_cast<const double2*>(row);
            const double2 km = *reinterpret_cast<const double2*>(sm_ + s * xrow);
            const double2 kp = *reinterpret_cast<const double2*>(sp_ + s * xrow);
            const double2 jm = *reinterpret_cast<const double2*>(row - N), jp = *reinterpret_cast<const double2*>(row + N);
            const double left = row[ileft];
            const double right = row[iright];
            lap[s].x = __dadd_rn(lap_plane(left, c2.y, jp.x, jm.x, c2.x), lap_z(kp.x, km.x, c2.x));
            lap[s].y = __dadd_rn(lap_plane(c2.x, right, jp.y, jm.y, c2.y), lap_z(kp.y, km.y, c2.y));
            xc[s] = c2;
          }
          double2 o0, o1;
          if (MODE & M_RESID) {
            bruss_resid(P, lap[0].x, lap[1].x, xc[0].x, xc[1].x, fo.x, o0.x, o1.x);
            bruss_resid(P, lap[0].y, lap[1].y, xc[0].y, xc[1].y, fo.y, o0.y, o1.y);
            if (MODE & M_NORM) nrm = fmax(nrm, fmax(fmax(abs_nf(o0.x), abs_nf(o0.y)), fmax(abs_nf(o1.x), abs_nf(o1.y))));
          } else {
            const double* yb = sc_ - N + 2 * xrow;   // the centre-only field of the same slot: [2][TS_L]
            const double2 y0 = *reinterpret_cast<const double2*>(yb);
            const double2 y1 = *reinterpret_cast<const double2*>(yb + TS_L);
            bruss_tangent<(MODE & M_VJP) != 0>(P, lap[0].x, lap[1].x, y0.x, y1.x, xc[0].x, xc[1].x, o0.x, o1.x);
            bruss_tangent<(MODE & M_VJP) != 0>(P, lap[0].y, lap[1].y, y0.y, y1.y, xc[0].y, xc[1].y, o0.y, o1.y);
          }
          double* dst = out + (int64_t)k * N2 + p;
          *reinterpret_cast<double2*>(dst) = o0;
          *reinterpret_cast<double2*>(dst + NC) = o1;
        }
        // done with the oldest plane (and, at the end of a march, with the other two).  Every consumer THREAD arrives: one elected
        // lane per warp after __syncwarp() is equivalent under the memory model but leaves compute-sanitizer's racecheck unable
        // to see that the other lanes' reads precede the producer's next copy into the slot
        mbar_arrive(&empty[sm_i]);
        if (jj + 1 == mc.m) { mbar_arrive(&empty[sc_i]); mbar_arrive(&empty[sp_i]); }
        sm_i = sc_i; sc_i = sp_i;
        if (++sp_i == R) { sp_i = 0; pp ^= 1; }
      }
    }
  }
  if (MODE & M_NORM) {
    nrm = block_max(nrm, red);
    if (threadIdx.x == 0) atomic_max_nonneg(norm_out, nrm);
  }
}

// ---- small analytic test problems
__device__ __forceinline__ double tri_apply(int64_t n, const double* x, int64_t i) {
  double s = 2.0 * x[i];
  if (i > 0) s -= x[i - 1];
  if (i + 1 < n) s -= x[i + 1];
  return s;
}
// kind: 0 quadratic, 1 tridiag.  what: M_RESID / M_JVP / M_VJP
__global__ void __launch_bounds__(PB_THREADS) small_problem_kernel(int kind, int what, int64_t n, double p, const double* __restrict__ pvec,
                                                                    const double* __restrict__ u, const double* __restrict__ d,
                                                                    double* __restrict__ out, double* __restrict__ norm_out) {
  __shared__ double red[32];
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  double nrm = 0.0;
  if (i < n) {
    double r;
    if (kind == 0) {
      if (what & M_RESID) r = u[i] * u[i] - p;
      else r = 2.0 * u[i] * d[i];
    } else {
      if (what & M_RESID) r = u[i] + 0.1 * u[i] * tri_apply(n, u, i) - pvec[i];
      else if (what & M_JVP) r = d[i] + 0.1 * (u[i] * tri_apply(n, d, i) + d[i] * tri_apply(n, u, i));
      else {  // J'w = w + 0.1 (T(u.*w) + (T u).*w)
        double t = 2.0 * u[i] * d[i];
        if (i > 0) t -= u[i - 1] * d[i - 1];
        if (i + 1 < n) t -= u[i + 1] * d[i + 1];
        r = d[i] + 0.1 * (t + tri_apply(n, u, i) * d[i]);
      }
    }
    out[i] = r;
    nrm = abs_nf(r);
  }
  if (what & M_NORM) {
    nrm = block_max(nrm, red);
    if (threadIdx.x == 0) atomic_max_nonneg(norm_out, nrm);
  }
}

__global__ void fd_eps_kernel(const double* dot_uv, double* eps_out) {
  // FiniteDiff.jl finite_difference_jvp!: eps = max(relstep * sqrt|x.v|, absstep), relstep = absstep = sqrt(eps(Float64))
  const double relstep = 1.4901161193847656e-08;
  *eps_out = fmax(relstep * sqrt(fabs(*dot_uv)), relstep);
}
__global__ void __launch_bounds__(PB_THREADS) fd_combine_kernel(int64_t n, const double* __restrict__ eps_ptr, const double* f1,
                                                                 const double* __restrict__ f0, double* out) {
  const double eps = *eps_ptr;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = (f1[i] - f0[i]) / eps;
}
__global__ void __launch_bounds__(PB_THREADS) fd_perturb_kernel(int64_t n, const double* __restrict__ eps_ptr, const double* __restrict__ u,
                                                                 const double* __restrict__ v, double* __restrict__ out) {
  const double eps = *eps_ptr;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = u[i] + eps * v[i];
}

__global__ void __launch_bounds__(PB_THREADS) bruss_u0_kernel(int dim, int N, int mode, double* __restrict__ u) {
  const int64_t NC = (dim == 2) ? (int64_t)N * N : (int64_t)N * N * N;
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= NC) return;
  const int i = (int)(c % N), j = (int)((c / N) % N), k = (int)(c / ((int64_t)N * N));
  const double x = (double)i / (double)(N - 1), y = (double)j / (double)(N - 1);
  double fac = 1.0;
  if (dim == 3 && mode == B200_U0_PERTURBED_Z) {
    const double z = (double)k / (double)(N - 1);
    fac = 1.0 + 0.01 * sin(2.0 * 3.14159265358979323846 * z);
  }
  u[c] = 22.0 * pow(y * (1.0 - y), 1.5) * fac;
  u[c + NC] = 27.0 * pow(x * (1.0 - x), 1.5) * fac;
}

inline int grid_for(int64_t n) { return (int)((n + PB_THREADS - 1) / PB_THREADS); }

// Which Brusselator kernel an op runs and with what grid.  `tiled`: the op has a ring-kernel instantiation (residual, residual
// + norm, JVP, VJP); `has_y`: its slots also carry the centre-only field (JVP, VJP).  ring_slots == 0 selects the plain kernel.
struct StencilPlan {
  int ring_slots, grid, max_marches;
  size_t slot_bytes;
};
StencilPlan stencil_plan(int dim, int N, bool tiled, bool has_y, int sm_count) {
  const int64_t NC = (dim == 2) ? (int64_t)N * N : (int64_t)N * N * N;
  const StencilPlan plain{0, grid_for(NC), 0, 0};
  const int N2 = N * N;
  if (dim == 2 || !tiled || N % 2 != 0 || N2 < TS_L + 2 * N) return plain;
  const size_t slot = sizeof(double) * (2 * (size_t)(TS_L + 2 * N) + (has_y ? 2 * TS_L : 0));
  // two CTAs per SM share the 227 KB; the depth of the ring is not what bounds a kernel this short (a few microseconds of
  // traffic at N = 100), so it stays at up to 8 slots
  const int R = (int)std::min<size_t>(TS_MAXR, (size_t)(100 * 1024) / slot);
  const int per_sm = 2;
  const int chunks = (N2 + TS_L - 1) / TS_L;
  const int64_t W = (int64_t)chunks * N;
  // one wave, two CTAs per SM; every CTA gets a run of >= 2 planes and crosses at most TS_MAXMARCH - 1 chunk boundaries
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(per_sm * (int64_t)sm_count, W / 2));
  if (R < 4 || (W + grid - 1) / grid > (int64_t)(TS_MAXMARCH - 1) * N) return plain;
  // CTA b marches over plane-chunks [W b / grid, W (b + 1) / grid): one march per chunk its run touches (the kernel's prologue)
  int max_marches = 0;
  for (int b = 0; b < grid; ++b) {
    const int64_t w0 = W * b / grid, w1 = W * (b + 1) / grid;
    if (w1 > w0) max_marches = std::max(max_marches, (int)((w1 - 1) / N - w0 / N + 1));
  }
  return StencilPlan{R, grid, max_marches, slot};
}

template <int MODE>
int32_t launch_bruss(b200_problem* p, const double* u, const double* d, double* du, double* Jd, double* norm_out, const double* eps) {
  b200_ctx* ctx = p->ctx;
  BrussParams P{p->N, p->a, p->A, p->B};
  const double* forcing = p->pvec;
  // algorithmic bytes: residual 2 Bv, JVP/VJP/FD-JVP 3 Bv, fused residual+JVP 4 Bv (DESIGN.md)
  const int kid = (MODE & M_RESID) && !(MODE & (M_JVP | M_VJP)) ? B200_KID_RESIDUAL : B200_KID_JVP;
  const double pbytes = 8.0 * (double)p->n * (((MODE & M_RESID) ? 2.0 : 0.0) + ((MODE & (M_JVP | M_VJP | M_FD)) ? ((MODE & M_RESID) ? 2.0 : 3.0) : 0.0));
  constexpr bool tiled = MODE == M_RESID || MODE == (M_RESID | M_NORM) || MODE == M_JVP || MODE == M_VJP;
  constexpr bool has_y = (MODE & (M_JVP | M_VJP)) != 0;
  const StencilPlan pl = stencil_plan(p->kind == B200_PROB_BRUSS2D ? 2 : 3, p->N, tiled, has_y, ctx->sm_count);
  if (p->kind == B200_PROB_BRUSS2D) {
    PLAUNCH(ctx, kid, pbytes, (bruss2d_kernel<MODE>), pl.grid, PB_THREADS, 0, P, u, d, forcing, du, Jd, norm_out, eps);
  } else {
    bool done = false;
    if constexpr (tiled) if (pl.ring_slots > 0) {
      const size_t smem = pl.slot_bytes * pl.ring_slots;
      CUDA_TRY(ctx, cudaFuncSetAttribute(bruss3d_ring_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      PLAUNCH(ctx, kid, pbytes, (bruss3d_ring_kernel<MODE>), pl.grid, TS_THREADS + 32, smem, P, pl.ring_slots, u, d, forcing, (MODE & M_RESID) ? du : Jd, norm_out);
      done = true;
    }
    if (!done) PLAUNCH(ctx, kid, pbytes, (bruss3d_kernel<MODE>), pl.grid, PB_THREADS, 0, P, u, d, forcing, du, Jd, norm_out, eps);
  }
  CHECK_LAUNCH(ctx);
  return B200_OK;
}

int32_t create_common(b200_ctx* ctx, b200_problem** out, int32_t kind, int32_t N, int64_t n) {
  if (!ctx || !out) return B200_ERR_INVALID;
  b200_problem* p = new b200_problem();
  memset(p, 0, sizeof(*p));
  p->ctx = ctx;
  p->kind = kind;
  p->N = N;
  p->n = n;
  *out = p;
  return B200_OK;
}

int32_t create_bruss(b200_ctx* ctx, int dim, int32_t N, double A, double B, double alpha, b200_problem** out) {
  B200_REQUIRE(ctx, N >= 3 && (dim == 2 ? N <= 16384 : N <= 1024), "Brusselator grid size out of range (3 <= N)");
  const int64_t NC = (dim == 2) ? (int64_t)N * N : (int64_t)N * N * N;
  B200_TRY(create_common(ctx, out, dim == 2 ? B200_PROB_BRUSS2D : B200_PROB_BRUSS3D, N, 2 * NC));
  b200_problem* p = *out;
  p->A = A;
  p->B = B;
  p->alpha = alpha;
  const double dx = 1.0 / (double)(N - 1);  // step(range(0, stop = 1, length = N))
  p->a = alpha / (dx * dx);                 // alpha = alpha / dx^2   (sparsity_tests__item1.jl:15)
  // forcing plane brusselator_f(x_i, y_j) (sparsity_tests__item1.jl:10), z-independent; evaluated once on the host in
  // strict IEEE double with the reference's expression so that the mask is bit-identical to the reference's.
  std::vector<double> forcing((size_t)N * N);
  const double r2 = 0.1 * 0.1;
  for (int j = 0; j < N; ++j)
    for (int i = 0; i < N; ++i) {
      volatile double x = (double)i / (double)(N - 1), y = (double)j / (double)(N - 1);
      volatile double dx2 = (x - 0.3) * (x - 0.3), dy2 = (y - 0.6) * (y - 0.6);
      volatile double s = dx2 + dy2;
      forcing[(size_t)i + (size_t)N * j] = (s <= r2) ? 5.0 : 0.0;
    }
  double* dptr = nullptr;
  CUDA_TRY(ctx, cudaMalloc(&dptr, sizeof(double) * forcing.size()));
  CUDA_TRY(ctx, cudaMemcpyAsync(dptr, forcing.data(), sizeof(double) * forcing.size(), cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  p->pvec = dptr;
  return B200_OK;
}

int32_t ensure_fd_scratch(b200_problem* p, int copies) {
  if (!p->fd_scratch) CUDA_TRY(p->ctx, cudaMalloc(&p->fd_scratch, sizeof(double) * p->n * 2));
  (void)copies;
  return B200_OK;
}
}  // namespace

extern "C" {
int32_t b200_problem_create_bruss2d(b200_ctx* ctx, int32_t N, double A, double B, double alpha, b200_problem** prob) {
  B200_DEVICE_GUARD(ctx);
  return create_bruss(ctx, 2, N, A, B, alpha, prob);
}
int32_t b200_problem_create_bruss3d(b200_ctx* ctx, int32_t N, double A, double B, double alpha, b200_problem** prob) {
  B200_DEVICE_GUARD(ctx);
  return create_bruss(ctx, 3, N, A, B, alpha, prob);
}
int32_t b200_problem_create_quadratic(b200_ctx* ctx, int64_t n, double p, b200_problem** prob) {
  B200_DEVICE_GUARD(ctx);
  B200_REQUIRE(ctx, n > 0, "n must be positive");
  B200_TRY(create_common(ctx, prob, B200_PROB_QUADRATIC, 0, n));
  (*prob)->p = p;
  return B200_OK;
}
int32_t b200_problem_create_tridiag_quad(b200_ctx* ctx, int64_t n, const double* p_dev, b200_problem** prob) {
  B200_DEVICE_GUARD(ctx);
  B200_REQUIRE(ctx, n > 0 && p_dev, "n must be positive and p_dev non-null");
  B200_TRY(create_common(ctx, prob, B200_PROB_TRIDIAG_QUAD, 0, n));
  double* copy = nullptr;
  CUDA_TRY(ctx, cudaMalloc(&copy, sizeof(double) * n));
  CUDA_TRY(ctx, cudaMemcpyAsync(copy, p_dev, sizeof(double) * n, cudaMemcpyDeviceToDevice, ctx->stream));
  (*prob)->pvec = copy;
  return B200_OK;
}
int32_t b200_problem_create_callback(b200_ctx* ctx, int64_t n, b200_residual_cb f, b200_jvp_cb jvp, b200_jvp_cb vjp, void* user,
                                     b200_problem** prob) {
  B200_DEVICE_GUARD(ctx);
  B200_REQUIRE(ctx, n > 0 && f, "callback problem needs n > 0 and a residual callback");
  B200_TRY(create_common(ctx, prob, B200_PROB_CALLBACK, 0, n));
  (*prob)->f_cb = f;
  (*prob)->jvp_cb = jvp;
  (*prob)->vjp_cb = vjp;
  (*prob)->user = user;
  return B200_OK;
}
int32_t b200_problem_set_jac(b200_problem* prob, b200_jac_cb jac_dense, b200_jac_cb jac_nzval) {
  B200_DEVICE_GUARD(prob ? prob->ctx : nullptr);
  prob->jac_dense_cb = jac_dense;
  prob->jac_nzval_cb = jac_nzval;
  return B200_OK;
}
int32_t b200_problem_set_jac_prototype(b200_problem* prob, const int64_t* colptr, const int64_t* rowval, int32_t index_base) {
  B200_DEVICE_GUARD(prob ? prob->ctx : nullptr);
  b200_ctx* ctx = prob->ctx;
  B200_REQUIRE(ctx, colptr && rowval && (index_base == 0 || index_base == 1), "set_jac_prototype: bad arguments");
  const int64_t n = prob->n, nnz = colptr[n] - index_base;
  B200_REQUIRE(ctx, nnz >= 0 && colptr[0] == index_base, "set_jac_prototype: malformed column pointers");
  free(prob->proto_colptr); free(prob->proto_rowval);
  prob->proto_colptr = (int64_t*)malloc(sizeof(int64_t) * (n + 1));
  prob->proto_rowval = (int64_t*)malloc(sizeof(int64_t) * (nnz > 0 ? nnz : 1));
  for (int64_t c = 0; c <= n; ++c) prob->proto_colptr[c] = colptr[c] - index_base;
  for (int64_t e = 0; e < nnz; ++e) {
    prob->proto_rowval[e] = rowval[e] - index_base;
    if (prob->proto_rowval[e] < 0 || prob->proto_rowval[e] >= n) return ctx->fail(B200_ERR_INVALID, "set_jac_prototype: row index out of range", __FILE__, __LINE__);
  }
  return B200_OK;
}
int32_t b200_problem_destroy(b200_problem* p) {
  B200_DEVICE_GUARD(p ? p->ctx : nullptr);
  if (!p) return B200_OK;
  cudaStreamSynchronize(p->ctx->stream);
  if (p->kind != B200_PROB_CALLBACK && p->pvec) cudaFree(const_cast<double*>(p->pvec));
  if (p->fd_scratch) cudaFree(p->fd_scratch);
  free(p->proto_colptr); free(p->proto_rowval);
  delete p;
  return B200_OK;
}
int32_t b200_problem_n(b200_problem* p, int64_t* n) { *n = p->n; return B200_OK; }
int32_t b200_problem_set_AB(b200_problem* p, double A, double B) { p->A = A; p->B = B; return B200_OK; }

int32_t b200_problem_u0(b200_problem* p, int32_t mode, double* u) {
  B200_DEVICE_GUARD(p ? p->ctx : nullptr);
  b200_ctx* ctx = p->ctx;
  if (p->kind == B200_PROB_BRUSS2D || p->kind == B200_PROB_BRUSS3D) {
    const int dim = p->kind == B200_PROB_BRUSS2D ? 2 : 3;
    LAUNCH(ctx, bruss_u0_kernel, grid_for(p->n / 2), PB_THREADS, 0, dim, p->N, mode, u);
    CHECK_LAUNCH(ctx);
    return B200_OK;
  }
  return b200_fill(ctx, p->n, 1.0, u);
}

int32_t b200_residual(b200_problem* p, const double* u, double* du) {
  B200_DEVICE_GUARD(p ? p->ctx : nullptr);
  return b200i_residual_norm(p, u, du, nullptr);
}

int32_t b200_jvp(b200_problem* p, const double* u, const double* v, double* Jv) {
  B200_DEVICE_GUARD(p ? p->ctx : nullptr);
  b200_ctx* ctx = p->ctx;
  switch (p->kind) {
    case B200_PROB_BRUSS2D:
    case B200_PROB_BRUSS3D: return launch_bruss<M_JVP>(p, u, v, nullptr, Jv, nullptr, nullptr);
    case B200_PROB_QUADRATIC:
    case B200_PROB_TRIDIAG_QUAD:
      LAUNCH(ctx, small_problem_kernel, grid_for(p->n), PB_THREADS, 0, p->kind == B200_PROB_QUADRATIC ? 0 : 1, (int)M_JVP, p->n, p->p,
             p->pvec, u, v, Jv, nullptr);
      CHECK_LAUNCH(ctx);
      return B200_OK;
    case B200_PROB_CALLBACK:
      if (p->jvp_cb) B200_TRY(b200i_sync_for_callback(ctx));
      if (p->jvp_cb) return p->jvp_cb(p->user, u, v, Jv) == 0 ? B200_OK : ctx->fail(B200_ERR_CALLBACK, "jvp callback failed", __FILE__, __LINE__);
      return b200_jvp_fd(p, u, v, Jv);  // no jvp supplied: AutoFiniteDiff fallback (autodiff.jl:52-84 last resort)
  }
  return ctx->fail(B200_ERR_INVALID, "unknown problem kind", __FILE__, __LINE__);
}

int32_t b200_vjp(b200_problem* p, const double* u, const double* w, double* JTw) {
  B200_DEVICE_GUARD(p ? p->ctx : nullptr);
  b200_ctx* ctx = p->ctx;
  switch (p->kind) {
    case B200_PROB_BRUSS2D:
    case B200_PROB_BRUSS3D: return launch_bruss<M_VJP>(p, u, w, nullptr, JTw, nullptr, nullptr);
    case B200_PROB_QUADRATIC:
    case B200_PROB_TRIDIAG_QUAD:
      LAUNCH(ctx, small_problem_kernel, grid_for(p->n), PB_THREADS, 0, p->kind == B200_PROB_QUADRATIC ? 0 : 1, (int)M_VJP, p->n, p->p,
             p->pvec, u, w, JTw, nullptr);
      CHECK_LAUNCH(ctx);
      return B200_OK;
    case B200_PROB_CALLBACK:
      if (p->vjp_cb) B200_TRY(b200i_sync_for_callback(ctx));
      if (p->vjp_cb) return p->vjp_cb(p->user, u, w, JTw) == 0 ? B200_OK : ctx->fail(B200_ERR_CALLBACK, "vjp callback failed", __FILE__, __LINE__);
      return ctx->fail(B200_ERR_UNSUPPORTED, "callback problem has no vjp", __FILE__, __LINE__);
  }
  return ctx->fail(B200_ERR_INVALID, "unknown problem kind", __FILE__, __LINE__);
}

int32_t b200_residual_norminf(b200_problem* p, const double* u, double* du, double* norm_host) {
  B200_DEVICE_GUARD(p ? p->ctx : nullptr);
  b200_ctx* ctx = p->ctx;
  B200_REQUIRE(ctx, u && du && norm_host, "residual_norminf: bad arguments");
  CUDA_TRY(ctx, cudaMemsetAsync(ctx->d_scalars, 0, sizeof(double), ctx->stream));
  B200_TRY(b200i_residual_norm(p, u, du, ctx->d_scalars));
  B200_TRY(b200i_fetch_scalars(ctx, 1));
  *norm_host = ctx->h_scalars[0];
  return B200_OK;
}

int32_t b200_problem_stencil_plan(b200_problem* p, int32_t op, int32_t* ring_slots, int32_t* grid, int32_t* max_marches) {
  b200_ctx* ctx = p->ctx;
  B200_REQUIRE(ctx, p->kind == B200_PROB_BRUSS2D || p->kind == B200_PROB_BRUSS3D, "stencil_plan: not a Brusselator problem");
  B200_REQUIRE(ctx, op >= B200_STENCIL_RESIDUAL && op <= B200_STENCIL_VJP && ring_slots && grid && max_marches, "stencil_plan: bad arguments");
  const StencilPlan pl = stencil_plan(p->kind == B200_PROB_BRUSS2D ? 2 : 3, p->N, true, op == B200_STENCIL_JVP || op == B200_STENCIL_VJP, ctx->sm_count);
  *ring_slots = pl.ring_slots;
  *grid = pl.grid;
  *max_marches = pl.max_marches;
  return B200_OK;
}

int32_t b200_residual_jvp(b200_problem* p, const double* u, const double* v, double* du, double* Jv) {
  B200_DEVICE_GUARD(p ? p->ctx : nullptr);
  if (p->kind == B200_PROB_BRUSS2D || p->kind == B200_PROB_BRUSS3D) return launch_bruss<M_RESID | M_JVP>(p, u, v, du, Jv, nullptr, nullptr);
  B200_TRY(b200_residual(p, u, du));
  return b200_jvp(p, u, v, Jv);
}

// (f(u + eps v) - f(u)) / eps with FiniteDiff.jl's forward step; for the stencils both evaluations share one neighbourhood load.
int32_t b200_jvp_fd(b200_problem* p, const double* u, const double* v, double* Jv) {
  B200_DEVICE_GUARD(p ? p->ctx : nullptr);
  b200_ctx* ctx = p->ctx;
  double* d_dot = ctx->d_scalars + 8;
  double* d_eps = ctx->d_scalars + 9;
  B200_TRY(b200i_reduce_sum_dev(ctx, p->n, u, v, RED_DOT, d_dot));
  LAUNCH(ctx, fd_eps_kernel, 1, 1, 0, d_dot, d_eps);
  if (p->kind == B200_PROB_BRUSS2D || p->kind == B200_PROB_BRUSS3D) return launch_bruss<M_FD>(p, u, v, nullptr, Jv, nullptr, d_eps);
  B200_TRY(ensure_fd_scratch(p, 2));
  double* x1 = p->fd_scratch;
  double* f0 = p->fd_scratch + p->n;
  const int g = grid_for(p->n) > 2048 ? 2048 : grid_for(p->n);
  LAUNCH(ctx, fd_perturb_kernel, g, PB_THREADS, 0, p->n, d_eps, u, v, x1);
  B200_TRY(b200_residual(p, u, f0));
  B200_TRY(b200_residual(p, x1, Jv));
  LAUNCH(ctx, fd_combine_kernel, g, PB_THREADS, 0, p->n, d_eps, Jv, f0, Jv);
  CHECK_LAUNCH(ctx);
  return B200_OK;
}
}  // extern "C"

// residual with the ||f||_inf epilogue fused (K1 + K6: `evaluate_f!` utils.jl:200-207 + `maximum(abs, fu)` common_defaults.jl:37)
int32_t b200i_residual_norm(b200_problem* p, const double* u, double* du, double* d_norminf) {
  b200_ctx* ctx = p->ctx;
  switch (p->kind) {
    case B200_PROB_BRUSS2D:
    case B200_PROB_BRUSS3D:
      return d_norminf ? launch_bruss<M_RESID | M_NORM>(p, u, nullptr, du, nullptr, d_norminf, nullptr)
                       : launch_bruss<M_RESID>(p, u, nullptr, du, nullptr, nullptr, nullptr);
    case B200_PROB_QUADRATIC:
    case B200_PROB_TRIDIAG_QUAD:
      LAUNCH(ctx, small_problem_kernel, grid_for(p->n), PB_THREADS, 0, p->kind == B200_PROB_QUADRATIC ? 0 : 1,
             (int)(M_RESID | (d_norminf ? M_NORM : 0)), p->n, p->p, p->pvec, u, (const double*)nullptr, du, d_norminf);
      CHECK_LAUNCH(ctx);
      return B200_OK;
    case B200_PROB_CALLBACK:
      B200_TRY(b200i_sync_for_callback(ctx));
      if (p->f_cb(p->user, u, du) != 0) return ctx->fail(B200_ERR_CALLBACK, "residual callback failed", __FILE__, __LINE__);
      if (d_norminf) return b200i_reduce_sum_dev(ctx, p->n, du, nullptr, RED_MAXABS, d_norminf);
      return B200_OK;
  }
  return ctx->fail(B200_ERR_INVALID, "unknown problem kind", __FILE__, __LINE__);
}
