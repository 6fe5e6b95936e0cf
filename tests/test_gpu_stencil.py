"""GPU tests of the Brusselator stencil kernels (csrc/problems.cu) in every launch regime of the 3D halo-ring kernel and its
thread-per-cell fallback: each ring depth, one to four marches per CTA, the W / 2 grid, exact and ragged last chunks, chunks
shorter than a row, and every fallback cause an H100 reaches (odd N, small N, too shallow a ring).  The sizes come from the
launch-plan restatement of tests/test_stencil_plan.py at the context's SM count, and the library's own plan must agree with it.

Integer probes: with alpha = 2**k * dx * dx the coefficient a = alpha / dx^2 is exactly 2**k, so for integer A, B and states in
[-8, 8] every intermediate of the kernels (the forcing included) is an integer far below 2**53 and the outputs must equal an
int64 restatement bit for bit.  Rounded data is held to a per-cell bound of 16 units of roundoff on the sum of the absolute
terms, against a long-double restatement.  Above FULL_MAX the restatement runs on sampled planes (the first, last and
boundary planes of several CTAs' marches) and the device compares the whole output with an independent kernel."""
import ctypes as C

import numpy as np
import pytest

import nonlinearsolve_jl_b200 as nls
from test_stencil_plan import FAMILY_OP, OPS, TS_L, exact_alpha, family_sizes, forcing_plane, plan, ring_layout, select_sizes

pytestmark = pytest.mark.gpu

GUARD = 1024           # NaN-filled doubles on each side of every output
FULL_MAX = 160         # whole-field host restatement up to this N, sampled planes above
BLOCK_CELLS = 1 << 23  # cells per species in one upload block
SALT_U, SALT_V, SALT_W = 0x1234, 0xBEEF, 0x5151
ULP_BOUND = 16 * 2.0 ** -53
K_EXACT = 3            # a = 8


def L():
    return nls.abi.lib()


def chk(ctx, status):
    nls.abi.check(ctx.handle, status)


def problem(ctx, dim, N, A, B, alpha):
    f = nls.Brusselator3D(N) if dim == 3 else nls.Brusselator2D(N)
    return nls._DeviceProblem(ctx, nls.NonlinearProblem(f, None, (A, B, alpha), ctx=ctx))


def dev_equal(ctx, x, y):
    eq = C.c_int32(-1)
    chk(ctx, L().b200_equal(ctx.handle, x.n, x.ptr, y.ptr, C.byref(eq)))
    return eq.value == 1


def residual_jvp_into(ctx, dp, u, v, du, Jv):
    chk(ctx, L().b200_residual_jvp(dp.handle, u.ptr, v.ptr, du.ptr, Jv.ptr))


class Guarded:
    """An n-vector view inside a NaN-filled allocation with GUARD doubles on either side."""

    def __init__(self, ctx, n):
        self.n = n
        self.buf = ctx.empty(n + 2 * GUARD).fill(np.nan)
        self.v = self.buf.view(GUARD, n)
        self.guard_bits = self._guards()

    def _guards(self):
        return np.concatenate([self.buf.view(0, GUARD).to_host(), self.buf.view(GUARD + self.n, GUARD).to_host()]).view(np.uint64)

    def check(self):
        assert np.array_equal(self._guards(), self.guard_bits), "a kernel wrote outside its output"
        assert np.isfinite(self.v.norm(np.inf)), "a cell of the output was never written"
        return self.v


# ----------------------------------------------------------------------------- probes and the restatement
def probe(N, salt, ks, integer=True):
    """Planes ks of a 2-species field as [s, k, j, i]: integers in [-8, 8], or floats in [0.25, 4.25) with 53 random bits,
    from a hash of (i, j, k, s) that varies along every index, so no misplaced plane or neighbour holds the right value."""
    i = np.arange(N, dtype=np.uint64)[None, None, None, :]
    j = np.arange(N, dtype=np.uint64)[None, None, :, None]
    k = np.asarray(list(ks), dtype=np.uint64)[None, :, None, None]
    s = np.arange(2, dtype=np.uint64)[:, None, None, None]
    h = (i * np.uint64(0x9E3779B97F4A7C15)) ^ (j * np.uint64(0xC2B2AE3D27D4EB4F)) ^ (k * np.uint64(0x165667B19E3779F9))
    h = h ^ (s * np.uint64(0x27D4EB2F165667C5) + np.uint64(salt))
    h ^= h >> np.uint64(31)
    h *= np.uint64(0xBF58476D1CE4E5B9)
    h ^= h >> np.uint64(29)
    if integer:
        return (h % np.uint64(17)).astype(np.int64) - 8
    return (h >> np.uint64(11)).astype(np.float64) * 2.0 ** -51 + 0.25


def upload(ctx, N, gen, dim=3):
    """A device vector holding the field gen(planes) -> [s, k, j, i], uploaded in blocks of planes."""
    if dim == 2:
        return ctx.to_device(gen([0]).astype(np.float64).ravel())
    NC, P = N ** 3, N * N
    vec = ctx.empty(2 * NC)
    step = max(1, BLOCK_CELLS // P)
    for k0 in range(0, N, step):
        ks = range(k0, min(N, k0 + step))
        X = gen(ks).astype(np.float64)
        for s in range(2):
            vec.view(s * NC + k0 * P, len(ks) * P).copy_from_host(X[s].ravel())
    return vec


def planes(vec, N, ks, dim=3):
    if dim == 2:
        return vec.to_host().reshape(2, 1, N, N)
    NC, P = N ** 3, N * N
    if list(ks) == list(range(N)):
        return vec.to_host().reshape(2, N, N, N)
    return np.stack([np.stack([vec.view(s * NC + k * P, P).to_host().reshape(N, N) for k in ks]) for s in range(2)])


def _lap(X, dim):
    """Periodic Laplacian (times dx^2) of X = [s, planes k0-1 .. k1, j, i] (3D) or [s, 1, j, i] (2D), and the sum of the
    absolute values of its terms."""
    Cc = X[:, 1:-1] if dim == 3 else X
    nb = [np.roll(Cc, 1, -1), np.roll(Cc, -1, -1), np.roll(Cc, 1, -2), np.roll(Cc, -1, -2)]
    if dim == 3:
        nb += [X[:, 2:], X[:, :-2]]
    lap = sum(nb) - (2 * dim) * Cc
    mag = sum(abs(t) for t in nb) + (2 * dim) * abs(Cc)
    return lap, mag, Cc


def stencil_ref(op, N, k0, k1, A, B, a, gu, gd=None, dim=3, exact=True):
    """(out, bound) of op in residual / jvp / vjp on planes k0 .. k1 - 1 as [s, k, j, i]: int64 when exact (A, B, a integers),
    else long double with the per-cell error bound ULP_BOUND * sum|terms| of the double evaluation."""
    ext = [(k0 - 1) % N] + list(range(k0, k1)) + [k1 % N] if dim == 3 else [0]
    cv = (lambda x: x.astype(np.int64)) if exact else (lambda x: x.astype(np.longdouble))
    if exact:
        A_, B_, a_, A1 = int(A), int(B), int(a), int(A) + 1
        assert (A_, B_, a_) == (A, B, a)
    else:
        A_, B_, a_, A1 = np.longdouble(A), np.longdouble(B), np.longdouble(a), np.longdouble(A + 1.0)
    fo = cv(forcing_plane(N))[None]
    X = cv(gu(ext) if op == "residual" else gd(ext))
    lap, mag, Xc = _lap(X, dim)
    U = Xc if op == "residual" else cv(gu(ext[1:-1] if dim == 3 else ext))
    u, v = U[0], U[1]
    uuv = u * u * v
    if op == "residual":
        f0 = a_ * lap[0] + B_ + uuv - A1 * u + fo
        f1 = a_ * lap[1] + A_ * u - uuv
        b0 = a_ * mag[0] + abs(B_) + abs(uuv) + abs(A1 * u) + abs(fo)
        b1 = a_ * mag[1] + abs(A_ * u) + abs(uuv)
    else:
        d, e = Xc[0], Xc[1]
        uv2, uu = 2 * u * v, u * u
        j00, j01, j10, j11 = uv2 - A1, uu, A_ - uv2, -uu
        m00, m01, m10, m11 = abs(uv2) + abs(A1), uu, abs(A_) + abs(uv2), uu   # bounds of |j..| before rounding
        if op == "vjp":
            j01, j10, m01, m10 = j10, j01, m10, m01
        f0 = a_ * lap[0] + j00 * d + j01 * e
        f1 = a_ * lap[1] + j10 * d + j11 * e
        b0 = a_ * mag[0] + m00 * abs(d) + m01 * abs(e)
        b1 = a_ * mag[1] + m10 * abs(d) + m11 * abs(e)
    return np.stack([f0, f1]), (None if exact else ULP_BOUND * np.stack([b0, b1]))


def sample_planes(N, op, sm):
    """Planes 0, 1, N/2, N-2, N-1, and the first and last plane of every march of several ring CTAs."""
    ks = {0, 1, N // 2, N - 2, N - 1}
    if plan(3, N, op, sm)[0]:
        grid, W, ms = ring_layout(N, op, sm)
        multi = [b for b in range(grid) if len(ms[b]) > 1][:3]
        for b in {0, 1, grid // 2, grid - 1, *multi}:
            for _, ka, m, _ in ms[b]:
                ks |= {ka, ka + m - 1}
    return sorted(ks)


def compare(vec, op, N, ks, A, B, a, gu, gd=None, dim=3, exact=True, what=""):
    """Device output vec against the restatement on planes ks (whole blocks when ks is every plane)."""
    blocks = [(0, N)] if (dim == 2 or list(ks) == list(range(N))) else [(k, k + 1) for k in ks]
    got = planes(vec, N, [k for k0, k1 in blocks for k in range(k0, k1)] if dim == 3 else [0], dim)
    q = 0
    refmax = 0
    for k0, k1 in blocks:
        ref, bound = stencil_ref(op, N, k0, k1, A, B, a, gu, gd, dim, exact)
        g = got[:, q:q + ref.shape[1]]
        q += ref.shape[1]
        if exact:
            bad = np.argwhere(g != ref)
            assert bad.size == 0, "%s %s N=%d: %d cells differ, first [s,k,j,i]=%s (k0=%d) got %r want %r" % (
                what, op, N, len(bad), bad[0], k0, g[tuple(bad[0])], ref[tuple(bad[0])])
        else:
            err = abs(g.astype(np.longdouble) - ref)
            bad = np.argwhere(err > bound)
            assert bad.size == 0, "%s %s N=%d: %d cells over the bound, first %s err %r bound %r" % (
                what, op, N, len(bad), bad[0], err[tuple(bad[0])], bound[tuple(bad[0])])
        refmax = max(refmax, abs(ref).max())
    return got, refmax


# ----------------------------------------------------------------------------- the plan the library launches
def test_plan_matches_restatement(ctx):
    sm = ctx.sm_count()
    for N in range(3, 1025):
        dp = problem(ctx, 3, N, 3.4, 1.0, 10.0)
        for op in range(4):
            assert dp.stencil_plan(op) == plan(3, N, op, sm), (N, OPS[op], sm)
        del dp
    for N in (3, 4, 5, 33, 100, 1000, 4097):
        dp = problem(ctx, 2, N, 3.4, 1.0, 10.0)
        for op in range(4):
            assert dp.stencil_plan(op) == plan(2, N, op, sm)
    sel = select_sizes(sm)
    print("\nSM count %d; N per launch class:" % sm)
    for c in sorted(sel, key=lambda c: (sel[c], c)):
        print("  %-45s N = %d  plan %s" % (c, sel[c], plan(3, sel[c], FAMILY_OP.get(c[0], 0), sm)))


# ----------------------------------------------------------------------------- exact integer probes, every regime
def _exact_residual(ctx, sm, N):
    a = 2 ** K_EXACT
    n, full = 2 * N ** 3, N <= FULL_MAX
    ks = list(range(N)) if full else sample_planes(N, 0, sm)
    ring = plan(3, N, 0, sm)[0] > 0
    gu = lambda pl: probe(N, SALT_U, pl)  # noqa: E731
    dp = problem(ctx, 3, N, 3.0, 2.0, exact_alpha(N, K_EXACT))
    u = upload(ctx, N, gu)
    for A, B in ((3, 2), (-2, 5)):
        if (A, B) != (3, 2):
            dp.set_AB(A, B)
        out = Guarded(ctx, n)
        dp.residual(u, out.v)
        _, refmax = compare(out.check(), "residual", N, ks, A, B, a, gu, what="residual")
        out2 = Guarded(ctx, n)
        _, nrm = dp.residual_norminf(u, out2.v)
        out2.check()
        assert dev_equal(ctx, out.v, out2.v)
        if full:
            assert nrm == refmax
        else:
            assert nrm == out.v.norm(np.inf) and nrm >= refmax
        del out2
        if ring:   # the fused op always runs the thread-per-cell kernel: an independent evaluation of the whole field
            du, Jv = ctx.empty(n), ctx.empty(n)
            residual_jvp_into(ctx, dp, u, u, du, Jv)
            assert dev_equal(ctx, du, out.v), "ring residual != plain residual (N=%d)" % N
            compare(Jv, "jvp", N, ks, A, B, a, gu, gu, what="residual_jvp")
            del du, Jv
        del out


def _exact_tangent(ctx, sm, N):
    a = 2 ** K_EXACT
    n, full = 2 * N ** 3, N <= FULL_MAX
    ks = list(range(N)) if full else sample_planes(N, 2, sm)
    gu, gv, gw = (lambda pl: probe(N, SALT_U, pl)), (lambda pl: probe(N, SALT_V, pl)), (lambda pl: probe(N, SALT_W, pl))
    dp = problem(ctx, 3, N, 3.0, 2.0, exact_alpha(N, K_EXACT))
    u, v, w = upload(ctx, N, gu), upload(ctx, N, gv), upload(ctx, N, gw)
    for A, B in ((3, 2), (-2, 5)):
        if (A, B) != (3, 2):
            dp.set_AB(A, B)
        oj, ov = Guarded(ctx, n), Guarded(ctx, n)
        dp.jvp(u, v, oj.v)
        dp.vjp(u, w, ov.v)
        Jv, _ = compare(oj.check(), "jvp", N, ks, A, B, a, gu, gv, what="jvp")
        JTw, _ = compare(ov.check(), "vjp", N, ks, A, B, a, gu, gw, what="vjp")
        if full:   # w . (J v) == v . (J' w), exactly, in integers
            W_, V_ = probe(N, SALT_W, range(N)), probe(N, SALT_V, range(N))
            assert int((W_ * Jv.astype(np.int64)).sum()) == int((V_ * JTw.astype(np.int64)).sum())
        else:      # every partial sum is an integer below 2**53: the device dot products are exact too
            assert oj.v.dot(w) == v.dot(ov.v)
        du, Jf = Guarded(ctx, n), Guarded(ctx, n)
        residual_jvp_into(ctx, dp, u, v, du.v, Jf.v)
        compare(du.check(), "residual", N, ks, A, B, a, gu, what="residual_jvp")
        assert dev_equal(ctx, Jf.check(), oj.v), "jvp != residual_jvp's jvp (N=%d)" % N
        del oj, ov, du, Jf


@pytest.mark.parametrize("family", ["residual", "tangent"])
def test_exact_probes_every_regime(ctx, family):
    sm = ctx.sm_count()
    for N in family_sizes(sm, family):
        (_exact_residual if family == "residual" else _exact_tangent)(ctx, sm, N)


@pytest.mark.parametrize("N", [3, 4, 5, 33, 2049])
def test_exact_probes_2d(ctx, N):
    a = 2 ** K_EXACT
    n = 2 * N * N
    gu, gv = (lambda pl: probe(N, SALT_U, [7])), (lambda pl: probe(N, SALT_V, [7]))
    dp = problem(ctx, 2, N, 3.0, 2.0, exact_alpha(N, K_EXACT))
    u, v = upload(ctx, N, gu, dim=2), upload(ctx, N, gv, dim=2)
    for A, B in ((3, 2), (-2, 5)):
        if (A, B) != (3, 2):
            dp.set_AB(A, B)
        out = Guarded(ctx, n)
        _, nrm = dp.residual_norminf(u, out.v)
        _, refmax = compare(out.check(), "residual", N, [0], A, B, a, gu, dim=2, what="residual_norminf 2d")
        assert nrm == refmax
        for op, call in (("residual", lambda o: dp.residual(u, o)), ("jvp", lambda o: dp.jvp(u, v, o)), ("vjp", lambda o: dp.vjp(u, v, o))):
            o = Guarded(ctx, n)
            call(o.v)
            compare(o.check(), op, N, [0], A, B, a, gu, gv, dim=2, what="2d")
        du, Jv = Guarded(ctx, n), Guarded(ctx, n)
        residual_jvp_into(ctx, dp, u, v, du.v, Jv.v)
        compare(du.check(), "residual", N, [0], A, B, a, gu, dim=2, what="residual_jvp 2d")
        compare(Jv.check(), "jvp", N, [0], A, B, a, gu, gv, dim=2, what="residual_jvp 2d")


# ----------------------------------------------------------------------------- rounded data, one ring N per depth
PARAMS = [(3.4, 1.0, 10.0), (2.75, 1.5, 0.37)]


@pytest.mark.parametrize("family", ["residual", "tangent"])
def test_rounded_data_every_ring_depth(ctx, family):
    sm = ctx.sm_count()
    sel = select_sizes(sm)
    Ns = sorted({N for c, N in sel.items() if c[:2] == (family, "R")})
    assert len(Ns) == (5 if family == "residual" else 2)
    for N in Ns:
        n, full = 2 * N ** 3, N <= FULL_MAX
        op = FAMILY_OP[family]
        ks = list(range(N)) if full else sample_planes(N, op, sm)
        gu, gv = (lambda pl: probe(N, SALT_U, pl, integer=False)), (lambda pl: probe(N, SALT_V, pl, integer=False) - 2.25)
        u, v = upload(ctx, N, gu), upload(ctx, N, gv)
        for A, B, alpha in PARAMS:
            dp = problem(ctx, 3, N, A, B, alpha)
            a = alpha / ((1.0 / (N - 1)) * (1.0 / (N - 1)))
            du, Jv = ctx.empty(n), ctx.empty(n)
            residual_jvp_into(ctx, dp, u, v, du, Jv)
            if family == "residual":
                o = Guarded(ctx, n)
                dp.residual(u, o.v)
                compare(o.check(), "residual", N, ks, A, B, a, gu, exact=False, what="rounded")
                assert dev_equal(ctx, o.v, du), "residual != residual_jvp's residual (N=%d)" % N
            else:
                oj, ov = Guarded(ctx, n), Guarded(ctx, n)
                dp.jvp(u, v, oj.v)
                dp.vjp(u, v, ov.v)
                compare(oj.check(), "jvp", N, ks, A, B, a, gu, gv, exact=False, what="rounded")
                compare(ov.check(), "vjp", N, ks, A, B, a, gu, gv, exact=False, what="rounded")
                assert dev_equal(ctx, oj.v, Jv), "jvp != residual_jvp's jvp (N=%d)" % N
            del du, Jv
        del u, v


@pytest.mark.parametrize("N", [26, 100])
def test_3d_slices_equal_2d_on_the_ring(ctx, N):
    # z-independent data: every k-slice of the 3D result (ring kernels at these N) equals the 2D result bit for bit
    sm = ctx.sm_count()
    assert all(plan(3, N, op, sm)[0] > 0 for op in range(4))
    d2, d3 = problem(ctx, 2, N, 3.4, 1.0, 10.0), problem(ctx, 3, N, 3.4, 1.0, 10.0)
    rng = np.random.default_rng(N)
    u2 = d2.u0().to_host() + 0.1 * rng.standard_normal(2 * N * N)
    v2 = rng.standard_normal(2 * N * N)
    tile = lambda x: np.concatenate([np.tile(x[:N * N], N), np.tile(x[N * N:], N)])  # noqa: E731
    U2, V2, U3, V3 = ctx.to_device(u2), ctx.to_device(v2), ctx.to_device(tile(u2)), ctx.to_device(tile(v2))
    pairs = [(d2.residual(U2), d3.residual(U3)), (d2.residual_norminf(U2)[0], d3.residual_norminf(U3)[0]),
             (d2.jvp(U2, V2), d3.jvp(U3, V3)), (d2.vjp(U2, V2), d3.vjp(U3, V3))]
    for r2, r3 in pairs:
        r2, r3 = r2.to_host(), r3.to_host()
        for k in range(N):
            for s in range(2):
                assert np.array_equal(r3[s * N ** 3 + k * N * N: s * N ** 3 + (k + 1) * N * N], r2[s * N * N:(s + 1) * N * N]), (N, k, s)


# ----------------------------------------------------------------------------- the fused maximum(abs, f) epilogue
def _spike_cells(N, sm):
    """(k, p, s) cells to hold the maximum: the first cell, the last pair of the (ragged) last chunk, the first and last plane
    of a march of CTAs with several marches, and a cell of species 1."""
    P = N * N
    cells = [(0, 0, 0), (N - 1, P - 2, 0), (N // 2, P - 1, 0), (0, 0, 1), (N - 1, P - 1, 1)]
    if plan(3, N, 0, sm)[0]:
        grid, W, ms = ring_layout(N, 0, sm)
        multi = [b for b in range(grid) if len(ms[b]) > 1]
        for b in (multi[:1] + multi[-1:]):
            for c, ka, m, _ in ms[b]:
                p = min(P - 1, c * TS_L + 37)
                cells += [(ka, p, 0), (ka + m - 1, p, 1)]
    return cells


@pytest.mark.parametrize("which", ["two_marches", "three_marches", "four_marches"])
def test_norm_epilogue_finds_the_maximum_anywhere(ctx, which):
    sm = ctx.sm_count()
    N = select_sizes(sm)[("residual", "marches", {"two_marches": 2, "three_marches": 3, "four_marches": 4}[which])]
    A, B, a, t = 2, 1, 2 ** K_EXACT, 8
    NC, P = N ** 3, N * N
    dp = problem(ctx, 3, N, A, B, exact_alpha(N, K_EXACT))
    u, du = ctx.zeros(2 * NC), Guarded(ctx, 2 * NC)
    fo = forcing_plane(N).ravel()
    for k, p, s in _spike_cells(N, sm):
        spike = u.view(s * NC + k * P + p, 1)
        spike.copy_from_host(np.array([float(t)]))

        def gen(pl, k=k, p=p, s=s):
            X = np.zeros((2, len(pl), N, N), dtype=np.int64)
            for q, kk in enumerate(pl):
                if kk == k:
                    X[s, q].flat[p] = t
            return X
        _, nrm = dp.residual_norminf(u, du.v)
        far = (k + N // 2) % N
        _, near_max = compare(du.check(), "residual", N, sorted({(k - 1) % N, k, (k + 1) % N, far}), A, B, a, gen, what="spike")
        # every plane but the three around the spike equals plane `far`, and the spike cell itself holds the maximum
        own = abs(-(6 * a + A + 1) * t + B + fo[p]) if s == 0 else 6 * a * t
        assert nrm == near_max == own, (N, k, p, s, nrm, near_max, own)
        # a NaN in the same cell is never dropped: +inf
        spike.copy_from_host(np.array([np.nan]))
        _, nrm_nan = dp.residual_norminf(u, du.v)
        assert nrm_nan == np.inf, (N, k, p, s)
        spike.copy_from_host(np.array([0.0]))


@pytest.mark.parametrize("N", [66, 25])
def test_norm_epilogue_zero_and_repeatable(ctx, N):
    # alpha = 0 (a = 0) with u = B + forcing, v = A / u: every residual is exactly zero, so the norm must be 0.0
    fo = forcing_plane(N).ravel()
    A, B = 6.0, 1.0
    u2 = B + fo
    state = np.concatenate([np.tile(u2, N), np.tile(A / u2, N)])
    dp = problem(ctx, 3, N, A, B, 0.0)
    du = Guarded(ctx, state.size)
    _, nrm = dp.residual_norminf(ctx.to_device(state), du.v)
    assert nrm == 0.0 and du.check().norm(np.inf) == 0.0
    # repeated calls on an integer probe agree bit for bit
    dp = problem(ctx, 3, N, 3.0, 2.0, exact_alpha(N, K_EXACT))
    u = upload(ctx, N, lambda pl: probe(N, SALT_U, pl))
    first = None
    for _ in range(3):
        o = ctx.empty(2 * N ** 3)
        _, nrm = dp.residual_norminf(u, o)
        if first is None:
            first = (o, nrm)
        else:
            assert nrm == first[1] and dev_equal(ctx, o, first[0])
    assert first[1] == first[0].norm(np.inf)


# ----------------------------------------------------------------------------- finite-difference JVP (plain kernels)
@pytest.mark.parametrize("N", [26, 25])
def test_fd_jvp(ctx, po, N):
    rng = np.random.default_rng(N)
    for A, B, alpha in PARAMS:
        dp = problem(ctx, 3, N, A, B, alpha)
        P = po.OracleProblem.bruss3d(N, A, B, alpha)
        u = P.u0(1) + 0.1 * rng.standard_normal(P.n)
        v = rng.standard_normal(P.n)
        fd = dp.jvp(ctx.to_device(u), ctx.to_device(v), fd=True).to_host()
        ref = P.jvp_fd(u, v)
        assert np.abs(fd - ref).max() <= 1e-6 * np.abs(ref).max(), (N, A, B, alpha)
