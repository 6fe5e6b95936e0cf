"""The dense LU (`b200_getrf` / `b200_getrs`, csrc/dense.cu) in every blocking regime up to the benchmark's n = 32768.

`Schedule` restates the host-side plan of `b200_getrf`: the outer block NBO (the trailing GEMM's K), the outer steps and,
for every inner panel of 32 columns, the grid of the cooperative panel kernel (CTAs P, rows per CTA rpc, shared memory) and
the stream it runs on (the first outer panel on the context's stream, every later one as the look-ahead panel on the
high-priority aux stream).  The tests use it to choose sizes for the device they run on and to assert that each case
reaches the regime it is named for.

Only what every correct partial-pivoting LU satisfies is asserted, whatever order it sums in:
  * ipiv[k] in [k + 1, n], and max |L_ij| <= 1 exactly (L is scaled by the reciprocal pivot and rounding is monotone, so
    a wrong arg-max anywhere breaks it);
  * Higham's Theorem 9.3 probed with nonnegative vectors x:  |P A x - L (U x)| <= 3 gamma_n (|L| (|U| x) + |P A| x),
    in long double on the host (n <= 4100) or with float64 cuBLAS matrix-vector products on the GPU (n >= 16384);
  * against LAPACK (n <= 4100): a normwise probe residual at most 10x LAPACK's, and LAPACK's pivots up to the first
    column where LAPACK's own choice is ambiguous;
  * padding rows of ld > n untouched, and bit-identical results when the same input is factored twice.
Exact equality is used only where the construction makes every operation exact: ties of equal magnitude at the start
of a block of a block upper triangular matrix, and exactly zero columns.
"""
import ctypes as C

import numpy as np
import pytest

NBI, PS_MAX, PANEL_ROWS = 32, 160, 128   # inner panel width, CTA cap of the panel grid, rows per panel CTA it aims for
PANEL_SMEM_MAX = 160 * 1024              # the panel kernel's dynamic shared-memory opt-in
U = 2.0 ** -53
H100_SM = 132
TIE = 2.0                                # magnitude of the tied entries; the other entries of a tie column are in (-1, 1)
NPROBE = 4
DEVICE = "cuda"


def gamma(k):
    return k * U / (1.0 - k * U)


# ------------------------------------------------------------------------------------------------ the host schedule
def nbo(n):
    return 512 if n >= 16384 else 256


def panel_grid(m, sm, kbi=NBI):
    """(P, rpc, dynamic shared memory bytes) of `panel_coop_kernel` for an inner panel of m rows."""
    P = min(sm, PS_MAX, max(1, -(-m // PANEL_ROWS)))
    rpc = -(-m // P)
    P = -(-m // rpc)
    return P, rpc, 8 * kbi * (rpc | 1)


class Panel:
    def __init__(self, c0, kbi, n, sm, k0):
        self.c0, self.kbi, self.k0 = c0, kbi, k0
        self.m = n - c0
        self.P, self.rpc, self.smem = panel_grid(self.m, sm, kbi)
        self.last_rows = self.m - (self.P - 1) * self.rpc
        self.stream = "main" if k0 == 0 else "aux"
        self.capped = self.rpc > PANEL_ROWS

    def cta(self, row):
        return (row - self.c0) // self.rpc

    def __repr__(self):
        return "panel(c0=%d, kbi=%d, P=%d, rpc=%d, last CTA %d rows, %s stream)" % (self.c0, self.kbi, self.P, self.rpc, self.last_rows, self.stream)


class Schedule:
    """The outer steps (k0, kbo, kbn) and inner panels of b200_getrf for an n x n matrix on `sm` SMs."""

    def __init__(self, n, sm):
        self.n, self.sm, self.nbo = n, sm, nbo(n)
        self.outer, self.panels = [], []
        for k0 in range(0, n, self.nbo):
            kbo = min(self.nbo, n - k0)
            rest = n - k0 - kbo
            self.outer.append((k0, kbo, min(self.nbo, rest) if rest > 0 else 0))
            self.panels += [Panel(k0 + i0, min(NBI, kbo - i0), n, sm, k0) for i0 in range(0, kbo, NBI)]

    def panel(self, col):
        return next(p for p in self.panels if p.c0 <= col < p.c0 + p.kbi)


def capped_n(sm):
    """The capped-grid size: the first panels have more rows than PANEL_ROWS x (CTA cap); 17000 on an H100."""
    return PANEL_ROWS * min(sm, PS_MAX) + 104


def recomputed_n(sm):
    """Smallest n >= 128 x cap whose first panel's grid is recomputed below the cap (P < cap, rpc > 128); 16897 on an H100."""
    cap = min(sm, PS_MAX)
    for n in range(PANEL_ROWS * cap + 1, PANEL_ROWS * cap + 4096):
        P, rpc, _ = panel_grid(n, sm)
        if P < cap and rpc > PANEL_ROWS:
            return n
    return None


def test_schedule_matches_the_h100_numbers():
    sm = H100_SM
    assert (nbo(16383), nbo(16384)) == (256, 512)
    s = Schedule(16384, sm)
    assert s.nbo == 512 and (s.panels[0].P, s.panels[0].rpc) == (128, 128) and not any(p.capped for p in s.panels)
    assert panel_grid(16897, sm)[:2] == (131, 129) and recomputed_n(sm) == 16897
    assert capped_n(sm) == 17000
    s = Schedule(17000, sm)
    assert (s.panels[0].P, s.panels[0].rpc) == (132, 129)
    assert [p.c0 for p in s.panels if p.capped] == [0, 32, 64, 96]          # block starts below column 104 are capped
    assert s.outer[-1][:2] == (16896, 104) and s.outer[-2][2] == 104        # short last outer panel, also the last look-ahead
    assert [p.kbi for p in s.panels if p.k0 == 16896] == [32, 32, 32, 8]
    s = Schedule(32768, sm)
    p = s.panels[0]
    assert (s.nbo, p.P, p.rpc, p.last_rows) == (512, 132, 249, 149)
    assert max(q.smem for q in s.panels) == 8 * 32 * 249 <= PANEL_SMEM_MAX
    assert [q.stream for q in s.panels[:17]] == ["main"] * 16 + ["aux"]
    s = Schedule(1000, sm)                                                  # the small tie / zero-pivot size
    assert s.nbo == 256 and s.outer[-1] == (768, 232, 0) and s.panels[-1].kbi == 8 and s.panels[-1].P == 1
    assert (panel_grid(128, sm)[0], panel_grid(129, sm)[:2]) == (1, (2, 65))


# ------------------------------------------------------------------------------------------------ device plumbing
def _torch():
    return pytest.importorskip("torch")


def _getrf(nls, ctx, At, n, ld):
    """Factor the column-major matrix whose column j is At[j, :n] (At: n x ld, float64, CUDA) in place."""
    torch = _torch()
    ipiv = torch.zeros(n, dtype=torch.int64, device=DEVICE)
    info = C.c_int32(-1)
    torch.cuda.synchronize()
    nls.abi.check(ctx.handle, nls.abi.lib().b200_getrf(ctx.handle, n, At.data_ptr(), ld, ipiv.data_ptr(), C.byref(info)))
    ctx.sync()
    return ipiv, info.value


def _getrs(nls, ctx, LUt, n, ld, ipiv, Bt, nrhs, ldb):
    torch = _torch()
    torch.cuda.synchronize()
    nls.abi.check(ctx.handle, nls.abi.lib().b200_getrs(ctx.handle, n, nrhs, LUt.data_ptr(), ld, ipiv.data_ptr(), Bt.data_ptr(), ldb))
    ctx.sync()


def _generator(seed):
    torch = _torch()
    g = torch.Generator(device=DEVICE)
    g.manual_seed(seed)
    return g


def _gaussian(n, ld, seed):
    """n x ld tensor At (row j = column j of A, padding rows n..ld-1 hold sentinels around 1e300)."""
    torch = _torch()
    g = _generator(seed)
    At = torch.randn((n, ld), generator=g, dtype=torch.float64, device=DEVICE)
    if ld > n:
        At[:, n:] = 1e300 * (1.0 + torch.rand((n, ld - n), generator=g, dtype=torch.float64, device=DEVICE))
    return At


def _bits(t):
    torch = _torch()
    return t.contiguous().view(torch.int64)


def perm_from_ipiv(ipiv):
    """Row order of P A for LAPACK's interchanges (1-based ipiv): (P A)[k] = A[perm[k]]."""
    perm = np.arange(len(ipiv))
    for k, p in enumerate(np.asarray(ipiv) - 1):
        if p != k:
            perm[k], perm[p] = perm[p], perm[k]
    return perm


def _report(label, **kw):
    print("[dense-lu] %s: %s" % (label, ", ".join("%s=%s" % kv for kv in kw.items())))


# ------------------------------------------------------------------------------------------------ host checks (n <= 4100)
def _host_probe(A, LU, ipiv, X):
    """(r, bound, |L| (|U| X)) of Theorem 9.3 in long double for the probes X (n x k, nonnegative)."""
    ld = np.longdouble
    n = A.shape[0]
    L = np.tril(LU, -1).astype(ld)
    L[np.diag_indices(n)] = 1
    Uu = np.triu(LU).astype(ld)
    PA = A[perm_from_ipiv(ipiv)].astype(ld)
    Xl = X.astype(ld)
    r = PA @ Xl - L @ (Uu @ Xl)
    lux = np.abs(L) @ (np.abs(Uu) @ Xl)
    return r, 3 * ld(gamma(n)) * (lux + np.abs(PA) @ Xl), lux


def _assert_structure(LU, ipiv, n, label):
    k = np.arange(1, n + 1)
    assert np.all((ipiv >= k) & (ipiv <= n)), "%s: ipiv out of range at %s" % (label, np.flatnonzero((ipiv < k) | (ipiv > n))[:5])
    lmax = np.abs(np.tril(LU, -1)).max() if n > 1 else 0.0
    assert lmax <= 1.0, "%s: max |L| = %r > 1 (column %d)" % (label, lmax, int(np.abs(np.tril(LU, -1)).max(axis=0).argmax()))


def check_factor_host(A, LU, ipiv, info, rng, label, expect_info=0):
    """Every getrf check that needs the matrix on the host: structure, long-double probe bound, LAPACK."""
    from scipy.linalg import lapack
    n = A.shape[0]
    assert info == expect_info, "%s: info %d, expected %d" % (label, info, expect_info)
    _assert_structure(LU, ipiv, n, label)
    X = rng.random((n, NPROBE))
    r, bound, _ = _host_probe(A, LU, ipiv, X)
    bad = np.abs(r) > bound
    assert not bad.any(), "%s: probe bound exceeded at rows %s (ratio %.3g)" % (label, np.flatnonzero(bad.any(axis=1))[:8],
                                                                               float((np.abs(r) / np.where(bound > 0, bound, 1)).max()))
    lu_l, piv_l, info_l = lapack.dgetrf(np.asfortranarray(A))
    assert info_l == info, "%s: LAPACK info %d, ours %d" % (label, info_l, info)
    r_l, _, lux_l = _host_probe(A, lu_l, piv_l + 1, X)
    ours = np.abs(r).max(axis=0)
    ref = np.maximum(np.abs(r_l).max(axis=0), n * U * lux_l.max(axis=0) / 100)
    assert np.all(ours <= 10 * ref), "%s: normwise probe residual %s vs LAPACK %s" % (label, ours, ref)
    colmax = np.abs(np.tril(lu_l, -1)).max(axis=0) if n > 1 else np.zeros(1)
    amb = np.flatnonzero(colmax > 1 - 1e-8)
    k_amb = int(amb[0]) if amb.size else n
    diff = np.flatnonzero(ipiv[:k_amb] != piv_l[:k_amb] + 1)
    assert diff.size == 0, "%s: pivot differs from LAPACK's at column %d (first ambiguous column %d)" % (label, diff[0], k_amb)
    return {"probe_ratio": "%.3g" % float((np.abs(r) / np.where(bound > 0, bound, 1)).max()),
            "vs_lapack": "%.3g" % float((ours / np.maximum(np.abs(r_l).max(axis=0), 1e-300)).max()), "first_ambiguous_column": k_amb if k_amb < n else None}, piv_l + 1


def factor_twice_host(nls, ctx, At, n, ld, label, rng, expect_info=0):
    """Factor At twice on one context (bit-identical), check the padding and every host check; returns (LU, ipiv, LAPACK ipiv)."""
    torch = _torch()
    A = At[:, :n].T.cpu().numpy().copy()
    LU1 = At.clone()
    ipiv1, info1 = _getrf(nls, ctx, LU1, n, ld)
    LU2 = At.clone()
    ipiv2, info2 = _getrf(nls, ctx, LU2, n, ld)
    assert info1 == info2 and torch.equal(_bits(LU1), _bits(LU2)) and torch.equal(ipiv1, ipiv2), "%s: two factorisations differ" % label
    if ld > n:
        assert torch.equal(_bits(LU1[:, n:]), _bits(At[:, n:])), "%s: padding rows changed" % label
    LU, ipiv = LU1[:, :n].T.cpu().numpy(), ipiv1.cpu().numpy()
    rep, piv_l = check_factor_host(A, LU, ipiv, info1, rng, label, expect_info)
    _report(label, n=n, ld=ld, NBO=nbo(n), **rep)
    return LU, ipiv, piv_l


# ------------------------------------------------------------------------------------------------ device checks (n >= 16384)
def check_factor_device(A0t, LUt, ipiv, n, seed, label, blk=2048):
    """Structure, |L| <= 1 and the probe bound with float64 cuBLAS products over column blocks (no full triangular copy)."""
    torch = _torch()
    ip = ipiv.cpu().numpy()
    k = np.arange(1, n + 1)
    assert np.all((ip >= k) & (ip <= n)), "%s: ipiv out of range" % label
    X = torch.rand((n, NPROBE), generator=_generator(seed), dtype=torch.float64, device=DEVICE)
    z = lambda: torch.zeros((n, NPROBE), dtype=torch.float64, device=DEVICE)  # noqa: E731
    Ax, aAx, Ux, aUx = z(), z(), z(), z()
    lmax = 0.0
    for j0 in range(0, n, blk):
        j1 = min(n, j0 + blk)
        a = A0t[j0:j1, :n].T
        Ax += a @ X[j0:j1]
        aAx += a.abs() @ X[j0:j1]
        u = torch.triu(LUt[j0:j1, :n].T, diagonal=-j0)
        Ux += u @ X[j0:j1]
        aUx += u.abs() @ X[j0:j1]
    LUx, aLaUx = Ux.clone(), aUx.clone()
    for j0 in range(0, n, blk):
        j1 = min(n, j0 + blk)
        lo = torch.tril(LUt[j0:j1, :n].T, diagonal=-j0 - 1)
        LUx += lo @ Ux[j0:j1]
        lo.abs_()
        lmax = max(lmax, float(lo.max()))
        aLaUx += lo @ aUx[j0:j1]
    assert lmax <= 1.0, "%s: max |L| = %r > 1" % (label, lmax)
    perm = torch.from_numpy(perm_from_ipiv(ip)).to(DEVICE)
    r = Ax[perm] - LUx
    bound = 3 * gamma(n) * (aLaUx + aAx[perm])
    bad = r.abs() > bound
    ratio = float((r.abs() / torch.where(bound > 0, bound, torch.ones_like(bound))).max())
    assert not bool(bad.any()), "%s: probe bound exceeded at rows %s (ratio %.3g)" % (label, torch.nonzero(bad.any(dim=1))[:8, 0].tolist(), ratio)
    normwise = float(r.abs().max(dim=0).values.div(n * U * aLaUx.max(dim=0).values).max())
    return {"probe_ratio": "%.3g" % ratio, "normwise_residual_over_nu": "%.3g" % normwise}


def _small_between(nls, ctx, rng):
    """A small factorisation on the same context between two large ones (the exchange table is reset per call)."""
    torch = _torch()
    n = 129
    A = rng.standard_normal((n, n))
    At = torch.tensor(A.T.copy(), device=DEVICE)
    ipiv, info = _getrf(nls, ctx, At, n, n)
    check_factor_host(A, At.T.cpu().numpy(), ipiv.cpu().numpy(), info, rng, "n=129 between two large factorisations")


def factor_twice_device(nls, ctx, A0t, n, label, seed, LU1=None):
    """LU of A0t (kept; LU1, when given, holds a copy of it), a small factorisation, the same LU again: bit-identical; then
    the device checks."""
    torch = _torch()
    LU1 = A0t.clone() if LU1 is None else LU1
    ipiv1, info1 = _getrf(nls, ctx, LU1, n, n)
    assert info1 == 0, "%s: info %d" % (label, info1)
    _small_between(nls, ctx, np.random.default_rng(seed))
    LU2 = A0t.clone()
    ipiv2, info2 = _getrf(nls, ctx, LU2, n, n)
    same = info2 == 0 and torch.equal(_bits(LU1), _bits(LU2)) and torch.equal(ipiv1, ipiv2)
    del LU2
    assert same, "%s: two factorisations of the same input differ" % label
    return LU1, ipiv1, check_factor_device(A0t, LU1, ipiv1, n, seed, label)


# ------------------------------------------------------------------------------------------------ getrf: seeded Gaussian matrices
@pytest.mark.gpu
@pytest.mark.parametrize("n,ld", [(127, 127), (128, 128), (129, 129), (255, 255), (513, 517), (2049, 2056), (4100, 4100)])
def test_getrf_gaussian(nls, ctx, n, ld):
    s = Schedule(n, ctx.sm_count())
    assert s.panels[0].P == (1 if n <= PANEL_ROWS else -(-n // PANEL_ROWS))
    factor_twice_host(nls, ctx, _gaussian(n, ld, seed=n), n, ld, "gaussian n=%d" % n, np.random.default_rng(n))


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["nbo512", "recomputed_grid", "capped_grid"])
def test_getrf_gaussian_large(nls, ctx, regime):
    sm = ctx.sm_count()
    n = {"nbo512": 16384, "recomputed_grid": recomputed_n(sm), "capped_grid": capped_n(sm)}[regime]
    if n is None:
        pytest.skip("no size recomputes the panel grid below the CTA cap on %d SMs" % sm)
    s = Schedule(n, sm)
    p = s.panels[0]
    cap = min(sm, PS_MAX)
    if regime == "nbo512":
        assert s.nbo == 512 and not any(q.capped for q in s.panels)
    elif regime == "recomputed_grid":
        assert p.P < cap and p.capped
    else:
        assert p.P == cap and p.capped and s.outer[-1][1] == n % s.nbo
    A0t = _gaussian(n, n, seed=n)
    _, _, rep = factor_twice_device(nls, ctx, A0t, n, "gaussian n=%d" % n, seed=n)
    _report("gaussian %s" % regime, n=n, NBO=s.nbo, first=p, last_outer=s.outer[-1], **rep)


@pytest.mark.gpu
def test_getrf_brusselator_n32768(nls, ctx, po):
    """The benchmark's own matrix: the dense Jacobian of the 2D Brusselator (N = 128) at u0, factored and solved."""
    torch = _torch()
    N = 128
    dp = nls._DeviceProblem(ctx, nls.NonlinearProblem(nls.Brusselator2D(N), None, (3.4, 1.0, 10.0), ctx=ctx))
    n = dp.n
    s = Schedule(n, ctx.sm_count())
    p = s.panels[0]
    assert n == 32768 and s.nbo == 512 and p.capped and p.P == min(ctx.sm_count(), PS_MAX)
    u = dp.u0()
    J = dp.dense_jacobian(u)                        # as bench.py's lu leg builds it, factored in place in its own buffer
    ctx.sync()
    Jt = torch.as_tensor(J, device=DEVICE).view(n, n)
    A0t = Jt.clone()
    torch.cuda.reset_peak_memory_stats()
    _, ipiv, rep = factor_twice_device(nls, ctx, A0t, n, "brusselator n=%d" % n, seed=n, LU1=Jt)
    b = dp.residual(u)
    x = b.copy()
    nls.abi.check(ctx.handle, nls.abi.lib().b200_getrs(ctx.handle, n, 1, J.ptr, n, ipiv.data_ptr(), x.ptr, n))
    xh, bh = x.to_host(), b.to_host()
    uh = u.to_host()                                 # the linearisation point J was filled at (the oracle's u0 may differ in the last bit)
    rel = np.abs(po.OracleProblem.bruss2d(N).jvp(uh, xh) - bh).max() / np.abs(bh).max()
    # Theorem 9.4: (J + dJ) x = f with |dJ| <= gamma_3n |L||U|, plus the rounding of the oracle's JVP and of its coefficients
    # (<= gamma_8 |J||x|), each with the factor 3 of the other bounds
    ax = torch.from_numpy(np.abs(xh)).to(DEVICE)
    lux, jx, uax = (torch.zeros(n, dtype=torch.float64, device=DEVICE) for _ in range(3))
    for j0 in range(0, n, 2048):
        j1 = min(n, j0 + 2048)
        uax += torch.triu(Jt[j0:j1].T, diagonal=-j0).abs() @ ax[j0:j1]
        jx += A0t[j0:j1].T.abs() @ ax[j0:j1]
    lux += uax
    for j0 in range(0, n, 2048):
        j1 = min(n, j0 + 2048)
        lux += torch.tril(Jt[j0:j1].T, diagonal=-j0 - 1).abs() @ uax[j0:j1]
    bound = 3 * (gamma(3 * n) * float(lux.max()) + gamma(8) * float(jx.max())) / np.abs(bh).max()
    _report("brusselator n=32768", NBO=s.nbo, first=p, solve_rel_residual="%.3g" % rel, solve_bound="%.3g" % bound,
            peak_GB="%.1f (torch) + %.1f (library J)" % (torch.cuda.max_memory_allocated() / 1e9, 8.0 * n * n / 1e9), **rep)
    assert rel <= bound, (rel, bound)


# ------------------------------------------------------------------------------------------------ exact cases
def _tie_rows(p, s, e, diag):
    """Rows of equal-magnitude entries for the block [s, e) whose first column lies in panel p: both sides of the first and of
    the last CTA boundary where they fall inside the block, the block's last row, and the diagonal row when asked."""
    rows = {e - 1}
    for k in sorted({1, p.P - 1}):
        b = p.c0 + k * p.rpc
        if 1 <= k < p.P and s <= b - 1 and b < e:
            rows |= {b - 1, b}
    if diag:
        rows.add(s)
    if len(rows) < 3 and e - s > 2:
        rows.add(s + 1 + (e - s - 1) // 2)
    return sorted(rows)


def tie_matrix(n, ld, starts, diag_starts, sm, seed):
    """Block upper triangular A (zero below the diagonal blocks) with block starts `starts`.  Elimination inside a block adds
    exact zeros to the rows below it, so the trailing column at every block start equals the original column in any correct
    implementation; that column gets tied maximal entries of mixed sign.  Returns (At, {start: (tie rows, panel)})."""
    torch = _torch()
    At = _gaussian(n, ld, seed)
    g = _generator(seed + 1)
    sched = Schedule(n, sm)
    bounds = list(starts) + [n]
    assert bounds[0] == 0 and all(a < b for a, b in zip(bounds, bounds[1:]))
    ties = {}
    for s, e in zip(bounds[:-1], bounds[1:]):
        At[s:e, e:n] = 0.0
        At[s, s:e] = 2.0 * torch.rand(e - s, generator=g, dtype=torch.float64, device=DEVICE) - 1.0
        p = sched.panel(s)
        rows = _tie_rows(p, s, e, s in diag_starts)
        At[s, rows] = torch.tensor([TIE if i % 2 == 0 else -TIE for i in range(len(rows))], dtype=torch.float64, device=DEVICE)
        ties[s] = (rows, p)
    return At, ties


def _tie_report(ties):
    return "; ".join("start %d: rows %s in CTAs %s of %r" % (s, rows, sorted({p.cta(r) for r in rows}), p) for s, (rows, p) in ties.items())


def _assert_ties(ipiv, ties, label, lapack_ipiv=None):
    for s, (rows, p) in ties.items():
        assert ipiv[s] == rows[0] + 1, "%s: block start %d pivots on row %d, expected %d (ties %s, %r)" % (label, s, ipiv[s] - 1, rows[0], rows, p)
        if lapack_ipiv is not None:
            assert lapack_ipiv[s] == rows[0] + 1, "%s: LAPACK pivots on row %d at block start %d" % (label, lapack_ipiv[s] - 1, s)


@pytest.mark.gpu
def test_getrf_ties_small(nls, ctx):
    """n = 1000 (NBO 256): block starts at column 0 (diagonal tie), inside an inner panel (45), at an inner-panel boundary
    (64), at the outer boundary that starts the first look-ahead panel (256, diagonal tie), at the next one (512) and in the
    narrow last panel (995 of [992, 1000))."""
    n, sm = 1000, ctx.sm_count()
    At, ties = tie_matrix(n, n, [0, 45, 64, 256, 512, 995], {0, 256}, sm, seed=11)
    _, ipiv, piv_l = factor_twice_host(nls, ctx, At, n, n, "ties n=%d" % n, np.random.default_rng(11))
    _assert_ties(ipiv, ties, "ties n=%d" % n, piv_l)
    assert ties[512][1].P > 2 and ties[512][1].cta(ties[512][0][-2]) == ties[512][1].P - 1  # a tie inside the last CTA
    _report("ties n=%d" % n, ties=_tie_report(ties))


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["many_blocks", "last_cta"])
def test_getrf_ties_capped(nls, ctx, layout):
    """n = 128 x cap + 104 (NBO 512 on an H100).  many_blocks: starts in the capped panels (0, 40, 96), at the outer
    boundary 512 (diagonal tie, first look-ahead panel), inside an aux-stream panel (1069) and in the narrow last panel.
    last_cta: the block from column 100 to the end straddles the boundary of the capped panel's last CTA."""
    sm = ctx.sm_count()
    n = capped_n(sm)
    s = Schedule(n, sm)
    if layout == "many_blocks":
        starts, diag = [0, 40, 96, s.nbo, 2 * s.nbo + 45, n - (n % NBI) + 3], {s.nbo}
    else:
        starts, diag = [0, 40, 100], {40}
    At, ties = tie_matrix(n, n, starts, diag, sm, seed=n + len(starts))
    label = "ties %s n=%d" % (layout, n)
    _, ipiv, rep = factor_twice_device(nls, ctx, At, n, label, seed=n + 1)
    _assert_ties(ipiv.cpu().numpy(), ties, label)
    assert ties[40][1].capped and ties[0][1].capped
    if layout == "last_cta":
        rows, p = ties[100]
        assert p.capped and p.cta(rows[-2]) == p.P - 1 and p.cta(rows[0]) == 0
    else:
        assert ties[n - (n % NBI) + 3][1].kbi == n % NBI and ties[s.nbo][1].stream == "aux"
    _report(label, ties=_tie_report(ties), **rep)


def zero_matrix(n, ld, zero_cols, seed):
    At = _gaussian(n, ld, seed)
    for j in zero_cols:
        At[j, :n] = 0.0
    return At


def _assert_zero_cols(LU, ipiv, zero_cols, label):
    for j in zero_cols:
        assert ipiv[j] == j + 1, "%s: zero column %d pivots on row %d" % (label, j, ipiv[j] - 1)
        assert not np.any(LU[:, j]), "%s: column %d of the factors is not exactly zero" % (label, j)


@pytest.mark.gpu
@pytest.mark.parametrize("zero_cols", [[5, 300, 995], [300, 700], [995]])
def test_getrf_zero_pivots_small(nls, ctx, zero_cols):
    """n = 1000: a zero column in the first panel (context stream), in look-ahead panels (aux stream), in the narrow last panel."""
    n = 1000
    s = Schedule(n, ctx.sm_count())
    assert s.panel(5).stream == "main" and s.panel(300).stream == "aux" and s.panel(995).kbi == n % NBI
    label = "zero columns %s n=%d" % (zero_cols, n)
    LU, ipiv, _ = factor_twice_host(nls, ctx, zero_matrix(n, n, zero_cols, seed=sum(zero_cols)), n, n, label,
                                    np.random.default_rng(sum(zero_cols)), expect_info=zero_cols[0] + 1)
    _assert_zero_cols(LU, ipiv, zero_cols, label)
    _report(label, panels=[repr(s.panel(j)) for j in zero_cols])


@pytest.mark.gpu
@pytest.mark.parametrize("first", ["capped", "aux"])
def test_getrf_zero_pivots_capped(nls, ctx, first):
    """n = 128 x cap + 104: the first zero column in a capped panel (context stream) or in a look-ahead panel (aux stream)."""
    torch = _torch()
    sm = ctx.sm_count()
    n = capped_n(sm)
    s = Schedule(n, sm)
    zero_cols = [70, s.nbo + 88, n - 2] if first == "capped" else [s.nbo + 88, n - 2]
    assert s.panel(70).capped and s.panel(70).stream == "main" and s.panel(s.nbo + 88).stream == "aux"
    label = "zero columns %s n=%d" % (zero_cols, n)
    At = zero_matrix(n, n, zero_cols, seed=n + zero_cols[0])
    LU1 = At.clone()
    ipiv1, info1 = _getrf(nls, ctx, LU1, n, n)
    LU2 = At.clone()
    ipiv2, info2 = _getrf(nls, ctx, LU2, n, n)
    same = info1 == info2 and torch.equal(_bits(LU1), _bits(LU2)) and torch.equal(ipiv1, ipiv2)
    del LU2
    assert same, "%s: two factorisations differ" % label
    assert info1 == zero_cols[0] + 1, "%s: info %d" % (label, info1)
    ip = ipiv1.cpu().numpy()
    for j in zero_cols:
        assert ip[j] == j + 1 and not bool(LU1[j, :n].any()), "%s: zero column %d" % (label, j)
    rep = check_factor_device(At, LU1, ipiv1, n, n + 7, label)
    _report(label, info=info1, panels=[repr(s.panel(j)) for j in zero_cols], **rep)


# ------------------------------------------------------------------------------------------------ getrs
def _rhs(nrhs, n, ldb, B):
    """nrhs x ldb tensor (row r = right-hand side r), padding sentinels."""
    torch = _torch()
    Bt = torch.full((nrhs, ldb), -3.0e300, dtype=torch.float64, device=DEVICE)
    Bt[:, n:] += torch.arange(ldb - n, dtype=torch.float64, device=DEVICE) * 1e297
    Bt[:, :n] = torch.from_numpy(np.ascontiguousarray(B.T)).to(DEVICE)
    return Bt


def _solve_bound_check(L, Uu, perm, B, X, label):
    """Theorem 9.4 against the GPU's own factors, in long double: |P B - L U X| <= 3 gamma_3n |L| |U| |X|, column by column."""
    ldt = np.longdouble
    n = L.shape[0]
    Xl = X.astype(ldt)
    R = B[perm].astype(ldt) - L @ (Uu @ Xl)
    bound = 3 * ldt(gamma(3 * n)) * (np.abs(L) @ (np.abs(Uu) @ np.abs(Xl)))
    bad = np.abs(R) > bound
    ratio = float((np.abs(R) / np.where(bound > 0, bound, 1)).max())
    assert not bad.any(), "%s: solve bound exceeded in columns %s (ratio %.3g)" % (label, np.flatnonzero(bad.any(axis=0))[:8], ratio)
    return ratio


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 33, 1000, 2049])
def test_getrs(nls, ctx, n):
    torch = _torch()
    rng = np.random.default_rng(100 + n)
    lda = n + 3
    A = rng.standard_normal((n, n))
    LUt = torch.zeros((n, lda), dtype=torch.float64, device=DEVICE)
    LUt[:, :n] = torch.from_numpy(A.T.copy()).to(DEVICE)
    ipiv, info = _getrf(nls, ctx, LUt, n, lda)
    assert info == 0
    LU = LUt[:, :n].T.cpu().numpy()
    L = np.tril(LU, -1).astype(np.longdouble)
    L[np.diag_indices(n)] = 1
    Uu = np.triu(LU).astype(np.longdouble)
    perm = perm_from_ipiv(ipiv.cpu().numpy())
    ratios = {}
    for nrhs in (1, 3, 37):
        B = rng.standard_normal((n, nrhs))
        singles = np.empty((n, nrhs))
        for r in range(nrhs):
            Bt = _rhs(1, n, n, B[:, r:r + 1])
            _getrs(nls, ctx, LUt, n, lda, ipiv, Bt, 1, n)
            singles[:, r] = Bt[0].cpu().numpy()
        for ldb in (n, n + 7):
            label = "getrs n=%d nrhs=%d ldb=%d" % (n, nrhs, ldb)
            Bt = _rhs(nrhs, n, ldb, B)
            pad = Bt[:, n:].clone()
            _getrs(nls, ctx, LUt, n, lda, ipiv, Bt, nrhs, ldb)
            assert torch.equal(_bits(Bt[:, n:]), _bits(pad)), "%s: padding changed" % label
            X = Bt[:, :n].T.cpu().numpy()
            assert np.array_equal(X.view(np.int64), singles.view(np.int64)), \
                "%s: columns %s differ from single right-hand-side solves" % (label, np.flatnonzero((X != singles).any(axis=0))[:8])
        ratios[nrhs] = "%.3g" % _solve_bound_check(L, Uu, perm, B, singles, "getrs n=%d nrhs=%d" % (n, nrhs))
    _report("getrs n=%d" % n, lda=lda, bound_ratio=ratios)


@pytest.mark.gpu
def test_getrs_inverse_n300(nls, ctx):
    """nrhs = n: X = A^-1, as Broyden's true-Jacobian initialisation solves for it."""
    torch = _torch()
    n = 300
    A = np.random.default_rng(300).standard_normal((n, n))
    LUt = torch.from_numpy(A.T.copy()).to(DEVICE)
    ipiv, info = _getrf(nls, ctx, LUt, n, n)
    assert info == 0
    Bt = torch.eye(n, dtype=torch.float64, device=DEVICE)
    _getrs(nls, ctx, LUt, n, n, ipiv, Bt, n, n)
    X = Bt.T.cpu().numpy()
    for r in range(n):
        e = torch.zeros((1, n), dtype=torch.float64, device=DEVICE)
        e[0, r] = 1.0
        _getrs(nls, ctx, LUt, n, n, ipiv, e, 1, n)
        assert np.array_equal(e[0].cpu().numpy().view(np.int64), X[:, r].view(np.int64)), "column %d differs from its single solve" % r
    LU = LUt.T.cpu().numpy()
    L = np.tril(LU, -1).astype(np.longdouble)
    L[np.diag_indices(n)] = 1
    ratio = _solve_bound_check(L, np.triu(LU).astype(np.longdouble), perm_from_ipiv(ipiv.cpu().numpy()), np.eye(n), X, "getrs inverse n=300")
    _report("getrs inverse n=300", bound_ratio="%.3g" % ratio)


# ------------------------------------------------------------------------------------------------ the pivoted-QR rescue
def _linear_problem(nls, ctx, A, b):
    """F(u) = A u - b with a dense user jac! (column-major) and jvp, on the device through torch."""
    torch = _torch()
    n = A.shape[0]
    At, bt = torch.tensor(A, device=DEVICE), torch.tensor(b, device=DEVICE)

    def F(du, u, _p):
        torch.as_tensor(du, device=DEVICE).copy_(At @ torch.as_tensor(u, device=DEVICE) - bt)
        torch.cuda.synchronize()

    def JVP(Jv, v, u, _p):
        torch.as_tensor(Jv, device=DEVICE).copy_(At @ torch.as_tensor(v, device=DEVICE))
        torch.cuda.synchronize()

    def JAC(J, u, _p):
        torch.as_tensor(J, device=DEVICE).view(n, n).copy_(At.T)   # row c of the view = column c of J
        torch.cuda.synchronize()

    f = nls.NonlinearFunction(F, jvp=JVP, n=n, jac=JAC)
    return nls.NonlinearProblem(f, np.zeros(n), None, ctx=ctx)


def _singular(n, seed):
    """Gaussian with an exactly zero column and a column exactly twice another: rank n - 2."""
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((n, n))
    A[:, n // 3] = 0.0
    A[:, n - 2] = 2.0 * A[:, 1]
    return A, rng.standard_normal(n)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [37, 1100])
def test_qr_rescue(nls, ctx, n):
    """getrf reports info > 0 on a singular dense J; the Newton step then solves J x = F(u0) in the least-squares sense with
    the pivoted QR (one 1024-thread CTA: n = 1100 has more columns than threads).  With u0 = 0, x = u0 - u1 exactly."""
    A, b = _singular(n, n)
    rank = np.linalg.matrix_rank(A)
    assert rank == n - 2
    sol = nls.solve(_linear_problem(nls, ctx, A, b), nls.NewtonRaphson(), maxiters=1, termination_condition=nls.AbsNormTerminationMode())
    assert sol.retcode == nls.ReturnCode.MaxIters and sol.stats.nsteps == 1 and sol.stats.nfactors == 1, nls.ReturnCode.name(sol.retcode)
    x = -sol.u
    fu = -b                                                        # F(u0) at u0 = 0
    nnz = int(np.count_nonzero(x))
    assert nnz <= rank, "x has %d nonzeros, rank is %d" % (nnz, rank)
    assert x[n // 3] == 0.0
    xs = np.linalg.lstsq(A, fu, rcond=None)[0]
    res, res_min = np.linalg.norm(A @ x - fu), np.linalg.norm(A @ xs - fu)
    assert abs(res - res_min) <= 1e-10 * res_min, (res, res_min)
    _report("qr rescue n=%d" % n, rank=rank, nonzeros=nnz, residual=res, lstsq_residual=res_min)


@pytest.mark.gpu
def test_qr_rescue_not_offered_above_4096(nls, ctx):
    A, b = _singular(4097, 4097)
    sol = nls.solve(_linear_problem(nls, ctx, A, b), nls.NewtonRaphson(), maxiters=1, termination_condition=nls.AbsNormTerminationMode())
    assert sol.retcode == nls.ReturnCode.InternalLinearSolveFailed and sol.stats.nfactors == 1, nls.ReturnCode.name(sol.retcode)
