// mg_cell.cuh — the per-cell arithmetic of the geometric-multigrid V-cycle (mg.cu), shared by the launch-per-sweep cycle of
// mg.cu and the shared-memory cycle inside the batched ensemble kernel (ens_batched.cu), so that a trajectory's V-cycle in the
// ensemble kernel is bit-identical to the single-system preconditioner's.  Sharing the source is not enough for that: the
// compiler fuses a multiply and an add into one FMA where it sees fit, and it sees differently in the two kernels.  So every
// rounding is spelled out with the _rn intrinsics, which are never fused or split; they state the FMAs the plain expressions
// compiled to in mg.cu, whose machine code is unchanged by them.  The index type I is int64_t for device-wide grids and int for
// the per-CTA grids of the ensemble kernel (integer arithmetic only).
#pragma once
#include <stdint.h>

__device__ __forceinline__ int mg_wrap(int i, int N) { return i < 0 ? i + N : (i >= N ? i - N : i); }

template <typename I>
__device__ __forceinline__ void mg_cell_coords(I c, int N, int dim, int& i, int& j, int& k) {
  if (dim == 3) {
    const I N2 = (I)N * N;
    k = (int)(c / N2);
    const int r = (int)(c - (I)k * N2);
    j = r / N;
    i = r - j * N;
  } else {
    k = 0;
    j = (int)(c / N);
    i = (int)(c - (I)j * N);
  }
}

// One cell (both species) of the level operator and its 2x2 block-Jacobi smoother, at linearisation state `state`:
// MODE 0: out = A x ; 1: out = b - A x ; 2: out = x + omega D^-1 (b - A x) ; 3: out = omega D^-1 b  (x == 0)
template <int MODE, typename I>
__device__ __forceinline__ void mg_op_cell(I c, int N, int dim, I NC, double a, double A, const double* __restrict__ state,
                                           const double* __restrict__ x, const double* __restrict__ b, double* __restrict__ out,
                                           double omega) {
  // the 2x2 block D = [d00 d01; d10 d11] of the level operator: lapd = -2 dim a and uv2 = 2 uc vc enter unrounded
  const double uc = state[c], vc = state[c + NC];
  const double uc2 = __dadd_rn(uc, uc), uu = __dmul_rn(uc, uc);
  const double m2dim = -2.0 * dim;                          // exact
  const double t = __fma_rn(uc2, vc, -__dadd_rn(A, 1.0));  // uv2 - (A + 1)
  const double d10 = __fma_rn(-uc2, vc, A);                 // A - uv2
  const double d00 = __fma_rn(m2dim, a, t), d01 = uu, d11 = __fma_rn(m2dim, a, -uu);
  double r0, r1;
  if (MODE == 3) {
    r0 = b[c]; r1 = b[c + NC];
  } else {
    int i, j, k;
    mg_cell_coords(c, N, dim, i, j, k);
    const I N2 = (I)N * N;
    const I base = c - i;                   // start of the i-line
    const I cim = base + mg_wrap(i - 1, N), cip = base + mg_wrap(i + 1, N);
    const I jb = c - (I)j * N;              // same (i, k), j = 0
    const I cjm = jb + (I)mg_wrap(j - 1, N) * N, cjp = jb + (I)mg_wrap(j + 1, N) * N;
    const double x0 = x[c], x1 = x[c + NC];
    // x[cim] + x[cip] + x[cjp] + x[cjm] - 4 x0 (+ x[ckp] + x[ckm] - 2 x0 in 3D)
    double l0 = __fma_rn(x0, -4.0, __dadd_rn(__dadd_rn(__dadd_rn(x[cim], x[cip]), x[cjp]), x[cjm]));
    double l1 = __fma_rn(x1, -4.0, __dadd_rn(__dadd_rn(__dadd_rn(x[cim + NC], x[cip + NC]), x[cjp + NC]), x[cjm + NC]));
    if (dim == 3) {
      const I kb = c - (I)k * N2;
      const I ckm = kb + (I)mg_wrap(k - 1, N) * N2, ckp = kb + (I)mg_wrap(k + 1, N) * N2;
      l0 = __dadd_rn(l0, __dsub_rn(__dadd_rn(x[ckp], x[ckm]), __dadd_rn(x0, x0)));
      l1 = __dadd_rn(l1, __dsub_rn(__dadd_rn(x[ckp + NC], x[ckm + NC]), __dadd_rn(x1, x1)));
    }
    // a l0 + (uv2 - (A + 1)) x0 + uu x1 and a l1 + (A - uv2) x0 - uu x1: the problem's exact JVP, left to right
    const double y0 = __fma_rn(x1, uu, __fma_rn(x0, t, __dmul_rn(a, l0)));
    const double y1 = __fma_rn(x1, -uu, __fma_rn(x0, d10, __dmul_rn(a, l1)));
    if (MODE == 0) { out[c] = y0; out[c + NC] = y1; return; }
    r0 = __dsub_rn(b[c], y0); r1 = __dsub_rn(b[c + NC], y1);
    if (MODE == 1) { out[c] = r0; out[c + NC] = r1; return; }
  }
  // e = D^-1 r by Cramer's rule: det = d00 d11 - d01 d10, e0 = (d11 r0 - d01 r1) / det, e1 = (d00 r1 - d10 r0) / det
  const double det = __fma_rn(d00, d11, -__dmul_rn(d01, d10));
  const double e0 = __ddiv_rn(__fma_rn(r0, d11, -__dmul_rn(d01, r1)), det);
  const double e1 = __ddiv_rn(__fma_rn(r1, d00, -__dmul_rn(d10, r0)), det);
  if (MODE == 3) { out[c] = __dmul_rn(omega, e0); out[c + NC] = __dmul_rn(omega, e1); }
  else { out[c] = __fma_rn(e0, omega, x[c]); out[c + NC] = __fma_rn(e1, omega, x[c + NC]); }
}

// Vertex-centred transfers for any integer ratio r (coarse point I sits on fine point r I):
//   prolongation  fine[r I + d] = (1 - d/r) c[I] + (d/r) c[I + 1] per direction (multilinear)
//   restriction   R = P' / r^dim: coarse[I] = sum_{|d| < r} (1 - |d|/r)/r * fine[r I + d] per direction (r = 2: 1/4, 1/2, 1/4)
// Both species.  The sums run on one thread in a fixed order (no tree reduction), so every caller rounds alike.
template <typename I>
__device__ __forceinline__ void mg_restrict_cell(I C, int Nf, int Nc, int dim, int ratio, const double* __restrict__ fine,
                                                 double* __restrict__ coarse) {
  const I NCc = dim == 3 ? (I)Nc * Nc * Nc : (I)Nc * Nc;
  const I NCf = dim == 3 ? (I)Nf * Nf * Nf : (I)Nf * Nf;
  int cI, cJ, cK;
  mg_cell_coords(C, Nc, dim, cI, cJ, cK);
  double s0 = 0.0, s1 = 0.0;
  const int hi = ratio - 1;
  const int khi = dim == 3 ? hi : 0;
  const double rinv = 1.0 / ratio;
  // weight (1 - |d| / r) / r per direction, its product over the directions, and the sum, all in this order
  for (int dk = -khi; dk <= khi; ++dk) {
    const double wk = dim == 3 ? __dmul_rn(__fma_rn((double)abs(dk), -rinv, 1.0), rinv) : 1.0;
    const int fk = dim == 3 ? mg_wrap(ratio * cK + dk, Nf) : 0;
    for (int dj = -hi; dj <= hi; ++dj) {
      const double wj = __dmul_rn(__fma_rn((double)abs(dj), -rinv, 1.0), rinv);
      const int fj = mg_wrap(ratio * cJ + dj, Nf);
      for (int di = -hi; di <= hi; ++di) {
        const double w = __dmul_rn(__dmul_rn(wk, wj), __dmul_rn(__fma_rn((double)abs(di), -rinv, 1.0), rinv));
        const int fi = mg_wrap(ratio * cI + di, Nf);
        const I f = fi + (I)Nf * (fj + (I)Nf * fk);
        s0 = __fma_rn(w, fine[f], s0);
        s1 = __fma_rn(w, fine[f + NCf], s1);
      }
    }
  }
  coarse[C] = s0;
  coarse[C + NCc] = s1;
}

template <typename I>
__device__ __forceinline__ void mg_prolong_add_cell(I f, int Nf, int Nc, int dim, int ratio, const double* __restrict__ coarse,
                                                    double* __restrict__ fine) {
  const I NCc = dim == 3 ? (I)Nc * Nc * Nc : (I)Nc * Nc;
  const I NCf = dim == 3 ? (I)Nf * Nf * Nf : (I)Nf * Nf;
  int i, j, k;
  mg_cell_coords(f, Nf, dim, i, j, k);
  const double rinv = 1.0 / ratio;
  const int I0 = i / ratio, J0 = j / ratio, K0 = k / ratio;
  const int di = i - I0 * ratio, dj = j - J0 * ratio, dk = k - K0 * ratio;
  const int ni = di ? 2 : 1, nj = dj ? 2 : 1, nk = (dim == 3 && dk) ? 2 : 1;
  // weights d / r and 1 - d / r per direction (d / r rounded once and shared), their product, and the sum, in this order
  const double pi = __dmul_rn((double)di, rinv), pj = __dmul_rn((double)dj, rinv), pk = __dmul_rn((double)dk, rinv);
  double s0 = 0.0, s1 = 0.0;
  for (int ck = 0; ck < nk; ++ck) {
    const double wk = dim == 3 ? (ck ? pk : __dsub_rn(1.0, pk)) : 1.0;
    for (int cj = 0; cj < nj; ++cj) {
      const double wj = cj ? pj : __dsub_rn(1.0, pj);
      for (int ci = 0; ci < ni; ++ci) {
        const double w = __dmul_rn(__dmul_rn(wk, wj), ci ? pi : __dsub_rn(1.0, pi));
        const I C = mg_wrap(I0 + ci, Nc) + (I)Nc * (mg_wrap(J0 + cj, Nc) + (I)Nc * (dim == 3 ? mg_wrap(K0 + ck, Nc) : 0));
        s0 = __fma_rn(w, coarse[C], s0);
        s1 = __fma_rn(w, coarse[C + NCc], s1);
      }
    }
  }
  fine[f] = __dadd_rn(fine[f], s0);
  fine[f + NCf] = __dadd_rn(fine[f + NCf], s1);
}
