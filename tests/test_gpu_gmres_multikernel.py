"""The multi-kernel GMRES engine (csrc/gmres.cu: residual_init, init_finish, multidot, reduce_h, update, mgs_pass, givens,
normalize, backsolve and the host loop of b200_gmres_solve) in every streaming-grid regime.

Every streaming kernel gives CTA b the contiguous rows [b*chunk, (b+1)*chunk) of the n rows (chunk = ceil(n / G) rounded up to
even, `block_rows`); the per-CTA partial sums are then added by reduce_h (lanes of 32 over G) or by a 256-thread block sum over
G (init_finish, mgs_pass, givens).  `Geometry` restates the host's choice of G and of the row split, so that the tests pick, on
the device they run on, the n that reach each regime:

    regime            n (132 SMs)   G     what it reaches
    one CTA, odd      1023          1     the scalar tail row of every streaming kernel
    two CTAs, odd     1025          2     chunk 514, last CTA 511 rows
    G > 32            16 897        33    the lane loop of reduce_h wraps; last CTA 449 rows
    G > 256           131 585       257   the 256-stride partial loops wrap; the last CTA holds exactly one row
    G at the cap      270 337       528   chunk 514: CTA 525 has 487 rows, CTAs 526-527 are empty
    Brusselator cap   2 * 64^3      528   the built-in JVP under engine = "multikernel"

Three kinds of evidence:
  * exact probes: a weighted cyclic permutation A e_i = w_i e_sigma(i) with w_i = +-2^p and b = 2^q e_s.  Every quantity of
    the iteration is exact in double precision in any summation order (basis vectors are signed unit vectors, every h is 0 or
    +-2^p, every Givens rotation has c, s in {0, +-1}), so the Hessenberg matrix, the statistics and x are known bit for bit.
    The cycle's members sit in the first CTA, in the odd tail row, in the one-row CTA and on both sides of every chunk boundary;
  * the engine's own basis, captured: a callback operator receives V[k-1] itself, copies it to the host and applies the same
    library kernel as the native operator, so that the Arnoldi relation, orthonormality, the least-squares solution and the
    stopping step can be checked against float64 references within gamma_m bounds (the reference's own rounding included);
  * bit-identity relations between runs that must do the same arithmetic.
The implicit restart when the basis reaches GM_KCAP takes minutes and runs only with B200_SLOW_TESTS=1.  With -s the module
prints, at its end, the largest error-to-bound ratio of every invariant over the tests that ran.
"""
import ctypes as C
import math
import os
import time

import numpy as np
import pytest
import scipy.sparse as sp

U = 2.0 ** -53                       # unit roundoff of float64
GM_THREADS, RED_MAX_BLOCKS, GM_KCAP = 256, 2048, 16384
H100_SMS = 132
ORTHS = ("mgs", "cgs", "cgs2")
PASSES = {"mgs": 1, "cgs": 1, "cgs2": 2}


def gamma(m):
    return m * U / (1.0 - m * U)


# ----------------------------------------------------------------------------- geometry restatement (no GPU needed)
class Geometry:
    """Streaming grid of the multi-kernel engine for n rows on a device with `sm` SMs (b200_gmres_create, block_rows,
    the ew_grid of b200_gmres_solve and the grid of its residual / initial-norm launches)."""

    def __init__(self, n, sm):
        self.n, self.sm = n, sm
        self.G = min(4 * sm, max(1, n // 512))
        chunk = -(-n // self.G)
        self.chunk = chunk + (chunk & 1)
        starts = np.minimum(np.arange(self.G, dtype=np.int64) * self.chunk, n)
        ends = np.minimum(starts + self.chunk, n)
        self.rows = ends - starts
        self.nonempty = int((self.rows > 0).sum())
        self.empty = self.G - self.nonempty
        self.tail_rows = int(self.rows[self.nonempty - 1])
        self.ew_grid = min(-(-n // (2 * GM_THREADS)), 8 * sm)
        self.red_grid = min(self.G, RED_MAX_BLOCKS)

    def cta(self, row):
        return int(row) // self.chunk

    def boundaries(self):
        """First rows of CTAs 1 .. nonempty-1 (a boundary lies between row b*chunk - 1 and b*chunk)."""
        return [b * self.chunk for b in range(1, self.nonempty)]

    def describe(self, kmax=None):
        return "n=%d G=%d chunk=%d tail_rows=%d empty_ctas=%d%s" % (self.n, self.G, self.chunk, self.tail_rows, self.empty,
                                                                     "" if kmax is None else " max_k=%d" % kmax)


def regime_sizes(sm):
    """n of each regime on a device with `sm` SMs; None where the device cannot reach the regime (4 * sm too small)."""
    cap = 4 * sm
    return {"G1_odd": 1023, "G2_odd": 2 * 512 + 1, "G33": 33 * 512 + 1 if cap >= 33 else None,
            "G257_onerow": 257 * 512 + 1 if cap >= 257 else None, "Gcap_empty": cap * 512 + 1}


REGIMES = ("G1_odd", "G2_odd", "G33", "G257_onerow", "Gcap_empty")


def probe_cycles(geo, L_min=25, per_group=32, seed=0):
    """Cycles of exact probes for this geometry.  Every cycle holds a row of the first CTA (its start s), the last row n-1
    (the scalar tail row when n is odd, the single row of a one-row CTA) and both sides of up to `per_group` chunk boundaries;
    together the cycles cover every boundary.  Short cycles are padded with rows drawn from random non-empty CTAs.  The members
    are visited in a shuffled order, so consecutive basis vectors jump between CTAs; L_min = 25 leaves a remainder of the
    8-column groups of the update kernel."""
    rng = np.random.default_rng(seed)
    n = geo.n
    bnd = geo.boundaries()
    groups = [bnd[i:i + per_group] for i in range(0, len(bnd), per_group)] or [[]]
    cycles = []
    for g in groups:
        members = [3, n - 1]
        for r in g:
            members += [r - 1, r]
        members = list(dict.fromkeys(members))
        while len(members) < L_min:
            r = int(rng.integers(0, n))
            if r not in members:
                members.append(r)
        rest = members[1:]
        rng.shuffle(rest)
        cycles.append([members[0]] + rest)
    return cycles


# ----------------------------------------------------------------------------- exact permutation probes: expectations
class Probe:
    """A e_i = w_i e_sigma(i): sigma is the given cycle, the identity elsewhere (weight 1); b = 2^q e_s, s = cycle[0]."""

    def __init__(self, n, cycle, seed=0, q=3):
        rng = np.random.default_rng(seed + 7)
        self.n, self.cycle, self.L = n, list(cycle), len(cycle)
        self.sigma = np.arange(n, dtype=np.int64)
        self.w = np.ones(n)
        for a, b in zip(self.cycle, self.cycle[1:] + self.cycle[:1]):
            self.sigma[a] = b
        cyc = np.asarray(self.cycle)
        self.w[cyc] = rng.choice([-1.0, 1.0], self.L) * 2.0 ** rng.integers(-2, 3, self.L)
        self.s = self.cycle[0]
        self.beta = 2.0 ** q
        self.b = np.zeros(n)
        self.b[self.s] = self.beta
        # the exact iteration: v_j = sign_j e_{idx_j}
        L = self.L
        self.H = np.zeros((L + 1, L))
        idx, sign = self.s, 1.0
        for j in range(L):
            if j + 1 < L:
                self.H[j + 1, j] = abs(self.w[idx])
                sign *= np.sign(self.w[idx])
                idx = int(self.sigma[idx])
            else:
                self.H[0, j] = sign * self.w[idx]
        self.x = np.zeros(n)
        self.x[idx] = self.beta / self.H[0, L - 1] * sign
        self.last = idx

    def csc(self, ctx):
        return ("csc", ctx.to_device(np.arange(self.n + 1, dtype=np.int64), np.int64), ctx.to_device(self.sigma, np.int64), ctx.to_device(self.w), 0)

    def hraw(self, k, shift=0.0):
        """The capture layout (k + 1 entries per column) of the first k columns."""
        H = self.H.copy()
        for j in range(self.L):
            H[j, j] += shift
        return np.concatenate([H[:j + 2, j] for j in range(k)])


def test_geometry_restatement_pins_the_h100_regimes():
    """The restatement on a 132-SM H100 SXM, and the placement of the probes' cycle members."""
    table = {"G1_odd": (1023, 1, 1024, 1023, 0), "G2_odd": (1025, 2, 514, 511, 0), "G33": (16897, 33, 514, 449, 0),
             "G257_onerow": (131585, 257, 514, 1, 0), "Gcap_empty": (270337, 528, 514, 487, 2)}
    sizes = regime_sizes(H100_SMS)
    for name, (n, G, chunk, tail, empty) in table.items():
        geo = Geometry(sizes[name], H100_SMS)
        assert (geo.n, geo.G, geo.chunk, geo.tail_rows, geo.empty) == (n, G, chunk, tail, empty), (name, geo.describe())
        assert geo.red_grid == G and geo.ew_grid == min(-(-n // 512), 8 * H100_SMS)
        cycles = probe_cycles(geo)
        seen = set()
        for cyc in cycles:
            assert 20 <= len(cyc) <= 70 and len(set(cyc)) == len(cyc) and all(0 <= r < n for r in cyc)
            assert geo.cta(cyc[0]) == 0 and n - 1 in cyc                        # first CTA; odd tail row / one-row CTA
            assert all(geo.rows[geo.cta(r)] > 0 for r in cyc)                   # never an empty CTA
            seen |= set(cyc)
        for r in geo.boundaries():                                              # both sides of every chunk boundary
            assert r - 1 in seen and r in seen and geo.cta(r - 1) + 1 == geo.cta(r)
        if name in ("G33", "G257_onerow", "Gcap_empty"):
            assert any(geo.cta(r) >= 32 for r in seen)                          # reaches the wrapped lane of reduce_h
        if name in ("G257_onerow", "Gcap_empty"):
            assert any(geo.cta(r) >= 256 for r in seen)                         # and the wrapped 256-stride block sums
    assert Geometry(131585, H100_SMS).rows[256] == 1 and (Geometry(270337, H100_SMS).rows[525:] == [487, 0, 0]).all()
    assert Geometry(2 * 64 ** 3, H100_SMS).G == 528 and Geometry(16400, H100_SMS).G == 32
    # the probe's exact iteration: x solves A x = b
    pr = Probe(1025, probe_cycles(Geometry(1025, H100_SMS))[0])
    Ax = np.zeros(pr.n)
    np.add.at(Ax, pr.sigma, pr.w * pr.x)
    assert np.array_equal(Ax, pr.b)


# ============================================================================= GPU part
def _lib(nls):
    return nls.abi.lib()


def _check(nls, ctx, rc):
    nls.abi.check(ctx.handle, rc)


def _stats(st):
    return (st.status, st.iters, st.nmatvec, st.restarts, st.rnorm0, st.rnorm, st.tol)


class Spy:
    """A callback operator that records its operand (the engine's basis vector V[k-1]) and then applies `apply(x, y)`, a
    library kernel on device pointers; `nan_at` poisons the output of that call (1-based) at row `nan_row`."""

    def __init__(self, apply, nan_at=None, nan_row=0, keep_out=False):
        self.apply, self.V, self.Y, self.nan_at, self.nan_row, self.keep_out = apply, [], [], nan_at, nan_row, keep_out

    def __call__(self, y, x):
        self.V.append(x.to_host())
        self.apply(x, y)
        if self.nan_at is not None and len(self.V) == self.nan_at:
            y.view(self.nan_row, 1).copy_from_host(np.array([np.nan]))
        if self.keep_out:
            self.Y.append(y.to_host())


def _native_csc(nls, ctx, n, csc):
    _, cp, rv, nz, base = csc
    op = C.c_void_p()
    _check(nls, ctx, _lib(nls).b200_linop_from_csc(ctx.handle, n, cp.ptr, rv.ptr, nz.ptr, base, C.byref(op)))
    return op


def _apply_linop(nls, ctx, op):
    return lambda x, y: _check(nls, ctx, _lib(nls).b200_linop_apply(op, x.ptr, y.ptr))


def _solver(nls, ctx, n, orth, keep=0, **kw):
    return nls.GmresSolver(ctx, n, nls.KrylovJL_GMRES(orth=orth, engine="multikernel", **kw), atol=0.0, rtol=0.0, keep_hessenberg=keep)


def _hcount(k):
    return k * (k + 3) // 2


def _H_from_raw(raw, k):
    H = np.zeros((k + 1, k))
    off = 0
    for j in range(k):
        H[:j + 2, j] = raw[off:off + j + 2]
        off += j + 2
    return H


@pytest.fixture(scope="module")
def sizes(ctx):
    return regime_sizes(ctx.sm_count())


def _regime_n(sizes, name):
    n = sizes[name]
    if n is None:
        pytest.skip("%s: this device has too few SMs for the regime" % name)
    return n


# ----------------------------------------------------------------------------- §2 exact probes
def _run_probe(nls, ctx, pr, orth, k_expect, shift=0.0, **kw):
    keep = _hcount(pr.L + 2)
    gm = _solver(nls, ctx, pr.n, orth, keep=keep, **kw)
    csc = pr.csc(ctx)
    op = _native_csc(nls, ctx, pr.n, csc)
    if shift:
        _check(nls, ctx, _lib(nls).b200_linop_set_shift(op, shift))
    x, db = ctx.zeros(pr.n), ctx.to_device(pr.b)                 # held in names: a temporary is freed before the solve reads it
    st = nls.abi.GmresStats()
    try:
        _check(nls, ctx, _lib(nls).b200_gmres_solve(gm._h, op, db.ptr, x.ptr, C.byref(st)))
    finally:
        _lib(nls).b200_linop_destroy(op)
    H = gm.hessenberg(k_expect)[:_hcount(k_expect)] if k_expect > 0 else np.zeros(0)
    return x.to_host(), st, H


@pytest.mark.gpu
@pytest.mark.parametrize("orth", ORTHS)
@pytest.mark.parametrize("regime", REGIMES)
def test_exact_probe_every_regime(nls, ctx, sizes, regime, orth):
    n = _regime_n(sizes, regime)
    geo = Geometry(n, ctx.sm_count())
    for ci, cyc in enumerate(probe_cycles(geo)):
        # started in the first CTA, and in the last row: the one non-zero dot product of the run, h_1L = <v_1, A v_L>, lands in
        # the row of b (the odd tail row, the one-row CTA, the last non-empty CTA), the rest goes through the norms
        t = cyc.index(n - 1)
        for start, c in (("first CTA", cyc), ("row n-1", cyc[t:] + cyc[:t])):
            pr = Probe(n, c, seed=ci)
            x, st, H = _run_probe(nls, ctx, pr, orth, pr.L, itmax=pr.L + 2)
            where = "%s cycle %d from %s (%s; CTAs %s)" % (regime, ci, start, geo.describe(pr.L), sorted({geo.cta(r) for r in cyc}))
            assert np.array_equal(H, pr.hraw(pr.L)), where + ": Hessenberg column %d" % int(np.argmax(np.abs(_H_from_raw(H, pr.L) - pr.H).max(axis=0)))
            assert _stats(st) == (nls.abi.LS_SOLVED, pr.L, pr.L, 0, pr.beta, 0.0, 0.0), (where, _stats(st))
            assert np.array_equal(x, pr.x), where + ": x wrong at rows %s" % np.nonzero(x != pr.x)[0][:8]


@pytest.mark.gpu
@pytest.mark.parametrize("orth", ORTHS)
@pytest.mark.parametrize("regime", ("G2_odd", "G257_onerow"))
def test_exact_probe_restart_itmax_warm_start(nls, ctx, sizes, regime, orth):
    """Restart lengths that do and do not divide L, with check_every 1 / 3 / 8; itmax ending mid-cycle; a warm start at x*/2."""
    n = _regime_n(sizes, regime)
    geo = Geometry(n, ctx.sm_count())
    pr = Probe(n, probe_cycles(geo)[-1], seed=11)
    L = pr.L
    for m in (L, L + 3):                                        # the cycle fits: solved in the first cycle, no restart
        for ce in (1, 3, 8):
            x, st, H = _run_probe(nls, ctx, pr, orth, L, gmres_restart=m, check_every=ce, itmax=L + 2)
            assert _stats(st) == (nls.abi.LS_SOLVED, L, L, 0, pr.beta, 0.0, 0.0) and np.array_equal(x, pr.x), (regime, m, ce, _stats(st))
            assert np.array_equal(H, pr.hraw(L))
    divisor = next(d for d in range(5, L) if L % d == 0) if any(L % d == 0 for d in range(5, L)) else 5
    for m in sorted({divisor, 7, L - 1}):                      # GMRES(m < L) stagnates at x = 0 on a cyclic permutation
        T = 3 * m + 2
        for ce in (1, 3, 8):
            x, st, H = _run_probe(nls, ctx, pr, orth, m, gmres_restart=m, check_every=ce, itmax=T)
            restarts = -(-T // m) - 1
            assert _stats(st) == (nls.abi.LS_MAXITERS, T, T + restarts, restarts, pr.beta, pr.beta, 0.0), (regime, m, ce, _stats(st))
            assert not x.any()
            assert np.array_equal(H, pr.hraw(m))                 # every cycle restarts from b with x = 0: the same capture
    for T in (1, 5, L // 2, L - 1):                             # itmax mid-cycle: y = 0, rnorm = beta at every step
        for ce in (3, 8):
            x, st, H = _run_probe(nls, ctx, pr, orth, T, itmax=T, check_every=ce)
            assert _stats(st) == (nls.abi.LS_MAXITERS, T, T, 0, pr.beta, pr.beta, 0.0) and not x.any(), (regime, T, _stats(st))
            assert np.array_equal(H, pr.hraw(T))
    gm = nls.GmresSolver(ctx, n, nls.KrylovJL_GMRES(orth=orth, engine="multikernel", warm_start=True, itmax=L + 2), atol=0.0, rtol=0.0, keep_hessenberg=_hcount(L))
    x, st = gm.solve(pr.csc(ctx), ctx.to_device(pr.b), ctx.to_device(pr.x / 2))
    assert _stats(st) == (nls.abi.LS_SOLVED, L, L + 1, 0, pr.beta / 2, 0.0, 0.0) and np.array_equal(x.to_host(), pr.x), _stats(st)
    assert np.array_equal(gm.hessenberg(L)[:_hcount(L)], pr.hraw(L))      # r0 = b / 2: the same basis, the same H


@pytest.mark.gpu
def test_exact_probe_shifted_operator(nls, ctx, sizes):
    """b200_linop_set_shift: (A + sigma I) on a probe keeps every Hessenberg entry exact (h_jj = sigma), and x solves the
    shifted system."""
    n = _regime_n(sizes, "G257_onerow")
    geo = Geometry(n, ctx.sm_count())
    pr = Probe(n, probe_cycles(geo)[0], seed=3)
    sigma = 0.5
    x, st, H = _run_probe(nls, ctx, pr, "cgs2", pr.L, shift=sigma, itmax=pr.L)
    assert np.array_equal(H, pr.hraw(pr.L, shift=sigma))
    Asp = sp.csc_matrix((pr.w, pr.sigma, np.arange(n + 1)), shape=(n, n)) + sigma * sp.eye(n, format="csc")
    r = np.linalg.norm(pr.b - Asp @ x)
    assert st.status in (nls.abi.LS_SOLVED, nls.abi.LS_MAXITERS) and abs(r - st.rnorm) <= 1e-12 * pr.beta, (r, st.rnorm)


@pytest.mark.gpu
@pytest.mark.parametrize("orth", ORTHS)
def test_exact_probe_long_cycle(nls, ctx, orth):
    """A cycle of L = 300 through every chunk boundary of n = 16 400 rows (G = 32): the basis outgrows the small Krylov arrays
    three times (64 -> 128 -> 256 -> 512 columns: R, z, cs and sn are copied) and spans 19 slabs of 16 vectors."""
    n, L = 16400, 300
    geo = Geometry(n, ctx.sm_count())
    cyc = probe_cycles(geo, L_min=L, per_group=10 ** 9, seed=4)
    assert len(cyc) == 1 and len(cyc[0]) == L
    pr = Probe(n, cyc[0], seed=4)
    x, st, H = _run_probe(nls, ctx, pr, orth, L, itmax=L + 2)
    assert np.array_equal(H, pr.hraw(L)), geo.describe(L)
    assert _stats(st) == (nls.abi.LS_SOLVED, L, L, 0, pr.beta, 0.0, 0.0) and np.array_equal(x, pr.x), _stats(st)


@pytest.mark.gpu
@pytest.mark.skipif(os.environ.get("B200_SLOW_TESTS") != "1", reason="137 s on one H100 (700 W); set B200_SLOW_TESTS=1 to run it")
def test_exact_probe_implicit_restart_at_kcap(nls, ctx):
    """One cycle through all n = 16 400 rows, CGS: at k + 40 > GM_KCAP the basis cannot grow and b200_gmres_solve restarts
    implicitly from the current x, which is exactly 0 (y = 0 while the cycle is open); the second cycle ends on itmax = n.
    The only test of that branch; it takes 137 s on one H100 SXM at 700 W, so it runs on request (B200_SLOW_TESTS=1)."""
    n = 16400
    rng = np.random.default_rng(5)
    pr = Probe(n, [0] + list(rng.permutation(np.arange(1, n))), seed=5)
    gm = nls.GmresSolver(ctx, n, nls.KrylovJL_GMRES(orth="cgs", engine="multikernel"), atol=0.0, rtol=0.0)
    t0 = time.perf_counter()
    x, st = gm.solve(pr.csc(ctx), ctx.to_device(pr.b))
    print("GM_KCAP probe: %s, %.1f s" % (Geometry(n, ctx.sm_count()).describe(GM_KCAP - 40), time.perf_counter() - t0))
    assert (st.status, st.iters, st.restarts, st.nmatvec, st.rnorm) == (nls.abi.LS_MAXITERS, n, 1, n + 1, pr.beta), _stats(st)
    assert not x.to_host().any()


# ----------------------------------------------------------------------------- §3 the engine's own basis
RATIOS = {}


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    """At the end of the module: the largest error-to-bound ratio of each invariant over the tests that ran (shown with -s)."""
    yield
    for key, v in sorted(RATIOS.items()):
        print("ratio %-36s %.3e" % (key, v))


def _ratio(key, err, bound):
    r = float(np.max(np.asarray(err) / np.asarray(bound)))
    RATIOS[key] = max(RATIOS.get(key, 0.0), r)
    return r


def _random_sparse(n, seed, per_row=4):
    """Non-symmetric sparse operator with a controlled spectrum: diagonal in [1, 30] plus `per_row` off-diagonal entries per
    row of size 0.3 / sqrt(per_row) (Gershgorin discs well inside the right half plane)."""
    rng = np.random.default_rng(seed)
    d = np.exp(rng.uniform(0.0, np.log(30.0), n))
    rows = np.repeat(np.arange(n), per_row)
    cols = rng.integers(0, n, n * per_row)
    vals = rng.standard_normal(n * per_row) * (0.3 / math.sqrt(per_row))
    A = sp.csc_matrix((np.concatenate([d, vals]), (np.concatenate([np.arange(n), rows]), np.concatenate([np.arange(n), cols]))), shape=(n, n))
    A.sum_duplicates()
    A.sort_indices()
    return A


def _csc_device(ctx, A, base=0):
    return ("csc", ctx.to_device(A.indptr.astype(np.int64) + base, np.int64), ctx.to_device(A.indices.astype(np.int64) + base, np.int64),
            ctx.to_device(A.data.astype(np.float64)), base)


class HostOp:
    """float64 reference operator: y = A v and |A| |v|; `nnz_row` is its longest row (its rounding: gamma_{nnz_row})."""

    def __init__(self, matvec, absmatvec, nnz_row):
        self.mv, self.absmv, self.nnz_row = matvec, absmatvec, nnz_row


def _hostop_sparse(A):
    Aa, Ar = abs(A).tocsr(), A.tocsr()
    return HostOp(lambda v: Ar @ v, lambda v: Aa @ np.abs(v), int(np.diff(Ar.indptr).max()))


def _hostop_dense(A):
    Aa = np.abs(A)
    return HostOp(lambda v: A @ v, lambda v: Aa @ np.abs(v), A.shape[1])


def check_operator_images(V, W, hop, label):
    """The device operator's images W_j of the captured v_j against the host operator: both round within gamma_{nnz_row}."""
    for j, (v, w) in enumerate(zip(V, W)):
        err = np.abs(w - hop.mv(v))
        bound = 2.0 * gamma(hop.nnz_row + 1) * hop.absmv(v) + np.finfo(float).tiny
        assert np.all(err <= bound), "%s: operator image %d, row %d" % (label, j + 1, int(np.argmax(err / bound)))
        _ratio("operator_image", err, bound)


def check_arnoldi(V, W, H, k, passes, n, label, orth_assert):
    """A v_j = sum_{i <= j+1} h_ij v_i for j < k and ||A v_k - V_k h_k|| = h_{k+1,k}, with W_j the engine's own image of v_j:
    the residual of column j is the rounding of the Gram-Schmidt update (passes * (j + 1) fused multiply-adds per row), of the
    normalisation and of the host's own evaluation of the relation.  Unit norms always.  Orthogonality max |(V_S' V - I)| over a
    sample S of columns: asserted at O(k u) for CGS2, recorded for MGS and CGS (whose loss grows as the residual falls)."""
    V = np.stack(V[:k], axis=1)
    habs = np.abs(H).sum(axis=0)
    Vmax = max(1.0, np.linalg.norm(V, axis=0).max())
    for j in range(k):
        bound = 2.0 * gamma(passes * (j + 2) + 4) * (np.linalg.norm(W[j]) + habs[j] * Vmax)
        if j + 1 < k:
            err = np.linalg.norm(W[j] - V[:, :j + 2] @ H[:j + 2, j])
        else:
            err = abs(np.linalg.norm(W[j] - V[:, :j + 1] @ H[:j + 1, j]) - H[j + 1, j])
        assert err <= bound, "%s: Arnoldi relation, column %d: %.3e > %.3e" % (label, j + 1, err, bound)
        _ratio("arnoldi_relation", err, bound)
    dn = np.abs(np.linalg.norm(V, axis=0) ** 2 - 1.0)
    nb = 2.0 * gamma(n + 8)
    assert dn.max() <= nb, "%s: basis vector %d is not of unit norm (%.3e)" % (label, int(dn.argmax()) + 1, dn.max())
    _ratio("unit_norm", dn, nb)
    S = np.unique(np.linspace(0, k - 1, min(k, 64)).astype(int))
    Gm = V[:, S].T @ V
    Gm[np.arange(len(S)), S] -= 1.0
    orth = float(np.abs(Gm).max())
    ob = gamma(n) + (k + 1) * gamma(n + 2 * k)
    if orth_assert:
        assert orth <= ob, "%s: orthogonality %.3e > %.3e" % (label, orth, ob)
        _ratio("orthogonality_cgs2", orth, ob)
    else:
        key = "orthogonality_loss_" + label.split()[0] + " (recorded)"
        RATIOS[key] = max(RATIOS.get(key, 0.0), orth)
    return V, orth, ob


def check_coefficients(V, W, H, k, orth, n, label):
    """Each stored coefficient is the dot product it stands for.  CGS: h_ij = <v_i, A v_j>.  MGS: h_ij = <v_i, w_j^(i)>, with
    w_j^(i) = A v_j - sum_{l<i} h_lj v_l restated on the host from the stored coefficients (the device forms it with one fused
    multiply-add per term, the host with two roundings: they differ by at most gamma_{3i+1} (|A v_j| + sum_{l<i} |h_lj| |v_l|)
    per row).  Bound: the device's and the host's dot-product rounding, gamma_n |v_i|'|w|, plus |v_i|' times that difference.
    (The Arnoldi relation holds for whatever coefficients the update used; this is what sees a wrong dot product.)  Every
    column when n k^2 is small, else 12 of them."""
    cols = range(k) if n * k * k <= 2e8 else np.unique(np.linspace(0, k - 1, 12).astype(int))
    for j in cols:
        Vj, h, w = V[:, :j + 1], H[:j + 1, j], W[j]
        if orth == "cgs":
            ref = Vj.T @ w
            bound = 2.0 * gamma(n) * (np.abs(Vj).T @ np.abs(w))
        else:
            zero = np.zeros((n, 1))
            Wi = w[:, None] - np.concatenate([zero, np.cumsum(Vj[:, :-1] * h[:-1], axis=1)], axis=1)
            E = np.abs(w)[:, None] + np.concatenate([zero, np.cumsum(np.abs(Vj[:, :-1]) * np.abs(h[:-1]), axis=1)], axis=1)
            E *= np.array([gamma(3 * i + 1) for i in range(j + 1)])[None, :]
            ref = np.einsum("ri,ri->i", Vj, Wi)
            bound = 2.0 * gamma(n) * np.einsum("ri,ri->i", np.abs(Vj), np.abs(Wi) + E) + np.einsum("ri,ri->i", np.abs(Vj), E)
        err = np.abs(h - ref)
        bound = bound + np.finfo(float).tiny
        assert np.all(err <= bound), "%s: coefficient h_%d,%d = %.17g, reference %.17g (bound %.3e)" % (
            label, int(np.argmax(err / bound)) + 1, j + 1, h[np.argmax(err / bound)], ref[np.argmax(err / bound)], bound[np.argmax(err / bound)])
        _ratio("coefficients_" + orth, err, bound)


def check_least_squares(V, H, k, beta, x, x0, rnorm, label):
    """min ||beta e1 - H y|| solved independently (NumPy) from the captured H: x = x0 + V y within a bound that carries
    kappa(H), rnorm = the LS residual.  Returns y and the LS residual."""
    e1 = np.zeros(k + 1)
    e1[0] = beta
    y = np.linalg.lstsq(H, e1, rcond=None)[0]
    rls = np.linalg.norm(e1 - H @ y)
    sv = np.linalg.svd(H, compute_uv=False)
    kap, Hn, yn = sv[0] / sv[-1], sv[0], np.linalg.norm(y)
    gk = gamma(6 * (k + 2))
    dy = 2.0 * gk * kap * (2.0 + kap * rls / (Hn * yn)) * yn                       # perturbation of y: device and NumPy
    xr = x0 + V @ y
    xb = math.sqrt(k) * dy + 2.0 * gamma(k + 2) * np.linalg.norm(np.abs(V) @ np.abs(y))
    ex = np.linalg.norm(x - xr)
    assert ex <= xb, "%s: x vs x0 + V y: %.3e > %.3e (kappa %.2e)" % (label, ex, xb, kap)
    _ratio("x_vs_x0_plus_Vy", ex, xb)
    rb = 2.0 * gk * (Hn * yn + beta) * (1.0 + kap)
    er = abs(rnorm - rls)
    assert er <= rb, "%s: rnorm %.17g vs LS residual %.17g" % (label, rnorm, rls)
    _ratio("rnorm_vs_ls_residual", er, rb)
    return y, rls


def _givens_history(H, beta):
    """|residual| after every step: the Givens QR of H restated in NumPy."""
    k = H.shape[1]
    R = H.copy()
    z = np.zeros(k + 1)
    z[0] = beta
    rho = []
    for j in range(k):
        a, bb = R[j, j], R[j + 1, j]
        r = math.hypot(a, bb)
        c, s = a / r, bb / r
        Rj, Rj1 = R[j, j:].copy(), R[j + 1, j:].copy()
        R[j, j:], R[j + 1, j:] = c * Rj + s * Rj1, -s * Rj + c * Rj1
        z[j], z[j + 1] = c * z[j], -s * z[j]
        rho.append(abs(z[j + 1]))
    return np.array(rho)


def check_true_residual(hop, b, x, y, W_norms, habs, passes, rnorm, orth, ob, k, label, orth_assert):
    """||b - A x|| against rnorm: to the orthogonality level (CGS2), or at most sqrt(k + 1) rnorm (MGS, CGS); plus the
    Arnoldi-relation residuals weighted by |y| and the rounding of A x and of the host's evaluation."""
    tr = np.linalg.norm(b - hop.mv(x))
    arn = sum(2.0 * gamma(passes * (j + 2) + 4) * (W_norms[j] + habs[j]) * abs(y[j]) for j in range(k))
    opr = 2.0 * gamma(hop.nnz_row + 2) * (np.linalg.norm(hop.absmv(x)) + np.linalg.norm(b))
    if orth_assert:
        err, bound = abs(tr - rnorm), (orth + ob) * math.sqrt(k + 1) * rnorm + arn + opr
    else:
        err, bound = max(0.0, tr - math.sqrt(k + 1) * rnorm), arn + opr
    assert err <= bound, "%s: true residual %.6e vs rnorm %.6e" % (label, tr, rnorm)
    if orth_assert:
        _ratio("true_residual_vs_rnorm", err, bound)


def check_captured_run(Vl, Wl, H, k, orth, n, label, hop, b, x, rnorm, x0=None):
    """Every §3 invariant of one captured run; returns the LS residual history (for the stopping-step check)."""
    check_operator_images(Vl[:k], Wl[:k], hop, label)
    V, orth_loss, ob = check_arnoldi(Vl, Wl, H, k, PASSES[orth], n, label, orth == "cgs2")
    if orth != "cgs2":
        check_coefficients(V, Wl, H, k, orth, n, label)
    x0 = np.zeros(n) if x0 is None else x0
    beta = np.linalg.norm(b - hop.mv(x0)) if x0.any() else np.linalg.norm(b)
    y, _ = check_least_squares(V, H, k, beta, x, x0, rnorm, label)
    check_true_residual(hop, b, x, y, [np.linalg.norm(w) for w in Wl[:k]], np.abs(H).sum(axis=0), PASSES[orth], rnorm, orth_loss, ob, k,
                        label, orth == "cgs2")
    return _givens_history(H, beta)


def _spy_run(nls, ctx, n, orth, apply, b, itmax, **kw):
    spy = Spy(apply, keep_out=True)
    gm = nls.GmresSolver(ctx, n, nls.KrylovJL_GMRES(orth=orth, engine="multikernel", itmax=itmax, **kw), atol=0.0, rtol=0.0,
                         keep_hessenberg=_hcount(itmax + 1))
    x, st = gm.solve(spy, ctx.to_device(b))
    H = _H_from_raw(gm.hessenberg(st.iters)[:_hcount(st.iters)], st.iters)
    return x.to_host(), st, H, spy


def _stopping_step(nls, ctx, n, orth, native, b, rho, label):
    """A tolerance halfway between two consecutive reference residuals (where they differ most, in the second half of the
    run): the engine stops exactly after that step, whatever its polling interval."""
    rho = np.asarray(rho)
    gaps = (rho[:-1] - rho[1:]) / rho[:-1]
    h = len(gaps) // 2
    j = int(np.argmax(gaps[h:])) + h                       # tolerance between rho[j] (step j + 1) and rho[j + 1] (step j + 2)
    tol = 0.5 * (rho[j] + rho[j + 1])
    assert rho[j] - tol > 1e-6 * tol and tol - rho[j + 1] > 1e-6 * tol, "%s: no clear gap between consecutive residuals" % label
    for ce in (1, 8):
        gm = nls.GmresSolver(ctx, n, nls.KrylovJL_GMRES(orth=orth, engine="multikernel", check_every=ce, itmax=len(rho) + 8), atol=tol, rtol=0.0)
        _, st = gm.solve(native, ctx.to_device(b))
        assert (st.status, st.iters) == (nls.abi.LS_SOLVED, j + 2), "%s: stopped at %d, reference step %d" % (label, st.iters, j + 2)


@pytest.mark.gpu
@pytest.mark.parametrize("orth", ORTHS)
@pytest.mark.parametrize("regime", REGIMES)
def test_captured_basis_sparse_every_regime(nls, ctx, sizes, regime, orth):
    n = _regime_n(sizes, regime)
    geo = Geometry(n, ctx.sm_count())
    K = 70
    A = _random_sparse(n, seed=n)
    csc = _csc_device(ctx, A)
    op = _native_csc(nls, ctx, n, csc)
    b = np.random.default_rng(n + 1).standard_normal(n)
    try:
        x, st, H, spy = _spy_run(nls, ctx, n, orth, _apply_linop(nls, ctx, op), b, K)
    finally:
        _lib(nls).b200_linop_destroy(op)
    label = "%s %s (%s)" % (orth, regime, geo.describe(st.iters))
    assert (st.status, st.iters, len(spy.V)) == (nls.abi.LS_MAXITERS, K, K), label
    rho = check_captured_run(spy.V, spy.Y, H, K, orth, n, label, _hostop_sparse(A), b, x, st.rnorm)
    _stopping_step(nls, ctx, n, orth, csc, b, rho, label)


ORACLE_COLS = 30


def _column_dev(h, href, k):
    """Per Hessenberg column (k + 1 entries each): max |h - href| relative to the column's largest entry."""
    out, off = [], 0
    for j in range(1, k + 1):
        sl = slice(off, off + j + 1)
        off += j + 1
        out.append(np.abs(h[sl] - href[sl]).max() / np.abs(href[sl]).max())
    return np.array(out)


@pytest.mark.gpu
@pytest.mark.parametrize("orth", ("mgs", "cgs2"))
@pytest.mark.parametrize("regime", REGIMES)
def test_hessenberg_vs_oracle_every_regime(nls, ctx, po, sizes, regime, orth):
    """The first 30 Hessenberg columns and x against the C oracle's GMRES (oracle/oracle.c) on the same CSC operator: an
    implementation independent of the engine.  The allowance is a multiple of how far the oracle itself moves under a
    rounding-level change: a reordering of its sums (1 thread against all threads, as in the N = 100 parity tests) and b with
    one ulp added to half of its entries (below the oracle's threading threshold the first leaves its sums unchanged, while
    MGS amplifies rounding to ~1e-10 by column 30 here), with a floor of 1e-11."""
    n = _regime_n(sizes, regime)
    geo = Geometry(n, ctx.sm_count())
    K = ORACLE_COLS
    A = _random_sparse(n, seed=n + 9)
    b = np.random.default_rng(n + 10).standard_normal(n)
    cnt = _hcount(K)
    code = {"mgs": po.ORTH_MGS, "cgs2": po.ORTH_CGS2}[orth]
    csc_host = (A.indptr.astype(np.int64), A.indices.astype(np.int64), A.data.astype(np.float64), 0)
    opts = po.default_gmres_opts(atol=0.0, rtol=0.0, orth=code, itmax=K)
    nthreads = po.get_threads()
    xo, so, ho = po.gmres(b, csc=csc_host, opts=opts, want_hessenberg=cnt)
    po.set_threads(1)
    try:
        x1, _, h1 = po.gmres(b, csc=csc_host, opts=opts, want_hessenberg=cnt)
    finally:
        po.set_threads(nthreads)
    bp = np.where(np.random.default_rng(n + 11).random(n) < 0.5, np.nextafter(b, np.inf), b)
    x2, _, h2 = po.gmres(bp, csc=csc_host, opts=opts, want_hessenberg=cnt)
    env = np.maximum.accumulate(np.maximum(_column_dev(h1, ho, K), _column_dev(h2, ho, K)))
    xenv = max(np.abs(x1 - xo).max(), np.abs(x2 - xo).max()) / np.abs(xo).max()
    gm = _solver(nls, ctx, n, orth, keep=cnt, itmax=K)
    x, st = gm.solve(_csc_device(ctx, A), ctx.to_device(b))
    label = "%s %s (%s)" % (orth, regime, geo.describe(K))
    assert (st.status, st.iters) == (so.status, so.iters) == (nls.abi.LS_MAXITERS, K), label
    dev = _column_dev(gm.hessenberg(K)[:cnt], ho[:cnt], K)
    bound = 30.0 * env + 1e-11
    assert np.all(dev <= bound), "%s: Hessenberg column %d off by %.3e (bound %.3e)" % (label, int(np.argmax(dev / bound)) + 1, dev.max(), bound[np.argmax(dev / bound)])
    _ratio("hessenberg_vs_oracle", dev, bound)
    ex = np.abs(x.to_host() - xo).max() / np.abs(xo).max()
    assert ex <= max(30.0 * xenv, 1e-9), (label, ex, xenv)
    assert abs(st.rnorm - so.rnorm) <= max(30.0 * env[-1], 1e-9) * so.rnorm and abs(st.rnorm0 - so.rnorm0) <= 1e-13 * so.rnorm0, (label, st.rnorm, so.rnorm)


@pytest.mark.gpu
@pytest.mark.parametrize("orth", ORTHS)
@pytest.mark.parametrize("n", (1025, 4097))
def test_captured_basis_dense(nls, ctx, n, orth):
    geo = Geometry(n, ctx.sm_count())
    rng = np.random.default_rng(n)
    A = np.eye(n) * 1.5 + rng.standard_normal((n, n)) / math.sqrt(n)
    dA = ctx.to_device(A.ravel(order="F"))
    b = rng.standard_normal(n)
    K = 60
    x, st, H, spy = _spy_run(nls, ctx, n, orth, lambda x, y: _check(nls, ctx, _lib(nls).b200_gemv(ctx.handle, 0, n, n, dA.ptr, n, x.ptr, y.ptr)), b, K)
    label = "%s dense (%s)" % (orth, geo.describe(st.iters))
    assert (st.status, st.iters) == (nls.abi.LS_MAXITERS, K), label
    rho = check_captured_run(spy.V, spy.Y, H, K, orth, n, label, _hostop_dense(A), b, x, st.rnorm)
    _stopping_step(nls, ctx, n, orth, ("dense", dA), b, rho, label)


@pytest.fixture(scope="module")
def bruss64(nls, ctx, po):
    N = 64
    f, P = nls.Brusselator3D(N), po.OracleProblem.bruss3d(N)
    dp = nls._DeviceProblem(ctx, nls.NonlinearProblem(f, None, (3.4, 1.0, 10.0), ctx=ctx))
    u = P.u0(1)
    return dp, P, u, ctx.to_device(u)


def _bruss_hostop(po, P, u):
    """The oracle's JVP as the host operator; |J| from the oracle's assembled Jacobian (8 entries per row)."""
    colptr, rowval = P.pattern(1)
    colors, nc = po.coloring_column(P.n, colptr, rowval, 1)
    J = sp.csc_matrix((P.sparse_jac(u, colptr, rowval, colors, nc, 1), rowval - 1, colptr - 1), shape=(P.n, P.n))
    Ja = abs(J).tocsr()
    return HostOp(lambda v: P.jvp(u, v), lambda v: Ja @ np.abs(v), 8)


@pytest.mark.gpu
@pytest.mark.parametrize("orth", ORTHS)
def test_captured_basis_brusselator_at_cap(nls, ctx, po, bruss64, orth):
    dp, P, u, du = bruss64
    n = P.n
    geo = Geometry(n, ctx.sm_count())
    b = P.residual(u)
    K = 60
    x, st, H, spy = _spy_run(nls, ctx, n, orth, lambda x, y: dp.jvp(du, x, out=y), b, K)
    label = "%s bruss3d N=64 (%s)" % (orth, geo.describe(st.iters))
    assert (st.status, st.iters) == (nls.abi.LS_MAXITERS, K), label
    rho = check_captured_run(spy.V, spy.Y, H, K, orth, n, label, _bruss_hostop(po, P, u), b, x, st.rnorm)
    _stopping_step(nls, ctx, n, orth, nls.JacobianOperator(dp, du), b, rho, label)


@pytest.mark.gpu
def test_captured_basis_long_beyond_shared_memory_default(nls, ctx):
    """k = 6160 > 6112: update_kernel and backsolve_kernel stage more than 48 KB of coefficients (the opt-in set at create
    time), the small Krylov arrays double several times (64 -> 8192 columns) and the basis spans hundreds of slabs."""
    n, K = 8192, 6160
    rng = np.random.default_rng(8192)
    # a cyclic shift plus a sparse perturbation: eigenvalues around the origin, so the residual decreases slowly and never
    # reaches zero within K steps
    shift = sp.csc_matrix((np.ones(n), (np.roll(np.arange(n), 1), np.arange(n))), shape=(n, n))
    P = _random_sparse(n, seed=8192)
    A = sp.csc_matrix(shift + 0.2 * (P - sp.diags(P.diagonal())))
    A.sort_indices()
    csc = _csc_device(ctx, A)
    op = _native_csc(nls, ctx, n, csc)
    b = rng.standard_normal(n)
    t0 = time.perf_counter()
    try:
        x, st, H, spy = _spy_run(nls, ctx, n, "cgs2", _apply_linop(nls, ctx, op), b, K)
    finally:
        _lib(nls).b200_linop_destroy(op)
    dt = time.perf_counter() - t0
    geo = Geometry(n, ctx.sm_count())
    print("long basis run: %s, %.1f s (captured run, host copies included)" % (geo.describe(st.iters), dt))
    assert (st.status, st.iters) == (nls.abi.LS_MAXITERS, K), _stats(st)
    label = "cgs2 long basis (%s)" % geo.describe(K)
    V = np.stack(spy.V, axis=1)
    del spy.V[:]
    W = np.stack(spy.Y, axis=1)
    del spy.Y[:]
    check_operator_images([V[:, j] for j in range(0, K, 97)], [W[:, j] for j in range(0, K, 97)], _hostop_sparse(A), label)
    # every column at once: R[:, j] = W_j - sum_{i <= j+1} h_ij v_i for j < K - 1 (H is upper Hessenberg)
    R = W[:, :K - 1] - V @ H[:K, :K - 1]
    Rn = np.linalg.norm(R, axis=0)
    habs = np.abs(H).sum(axis=0)
    m = 2 * (np.arange(K) + 2) + 4
    bound = 2.0 * (m * U / (1.0 - m * U)) * (np.linalg.norm(W, axis=0) + habs * max(1.0, np.linalg.norm(V, axis=0).max()))
    assert np.all(Rn <= bound[:-1]), "%s: Arnoldi relation fails at column %d" % (label, int(np.argmax(Rn / bound[:-1])) + 1)
    _ratio("arnoldi_relation_long", Rn, bound[:-1])
    lastc = abs(np.linalg.norm(W[:, K - 1] - V @ H[:K, K - 1]) - H[K, K - 1])
    assert lastc <= bound[-1]
    del W, R
    S = np.unique(np.linspace(0, K - 1, 64).astype(int))
    Gm = V[:, S].T @ V
    Gm[np.arange(len(S)), S] -= 1.0
    ob = gamma(n) + (K + 1) * gamma(n + 2 * K)
    assert np.abs(Gm).max() <= ob, (np.abs(Gm).max(), ob)
    _ratio("orthogonality_long", np.abs(Gm).max(), ob)
    check_least_squares(V, H, K, np.linalg.norm(b), x, np.zeros(n), st.rnorm, label)


# ----------------------------------------------------------------------------- §4 bit-identity relations
@pytest.mark.gpu
@pytest.mark.parametrize("orth", ORTHS)
@pytest.mark.parametrize("regime", ("G2_odd", "G33", "G257_onerow", "Gcap_empty"))
def test_bit_identity_relations(nls, ctx, sizes, regime, orth):
    """Spy (status polled every step) = native operator at check_every 1 / 3 / 8 (kernels enqueued after convergence change
    nothing); a repeated solve; a solve after a longer one on the same cache (stale slabs and R); x0 = 0 as a warm start."""
    n = _regime_n(sizes, regime)
    A = _random_sparse(n, seed=n + 5)
    csc = _csc_device(ctx, A)
    op = _native_csc(nls, ctx, n, csc)
    b = np.random.default_rng(n + 6).standard_normal(n)
    db = ctx.to_device(b)
    K = 40
    try:
        xs, sts, Hs, _ = _spy_run(nls, ctx, n, orth, _apply_linop(nls, ctx, op), b, K)
    finally:
        _lib(nls).b200_linop_destroy(op)
    gm_ref = nls.GmresSolver(ctx, n, nls.KrylovJL_GMRES(orth=orth, engine="multikernel", itmax=K), atol=0.0, rtol=0.0, keep_hessenberg=_hcount(K))
    for ce in (1, 3, 8):
        gm = nls.GmresSolver(ctx, n, nls.KrylovJL_GMRES(orth=orth, engine="multikernel", itmax=K, check_every=ce), atol=0.0, rtol=0.0, keep_hessenberg=_hcount(K))
        x, st = gm.solve(csc, db)
        assert _stats(st) == _stats(sts) and np.array_equal(x.to_host(), xs), (regime, orth, ce, _stats(st), _stats(sts))
        assert np.array_equal(_H_from_raw(gm.hessenberg(K)[:_hcount(K)], K), Hs)
    # convergence strictly inside a polling window (step 19 is no multiple of 3 or 8): a tolerance between the residuals
    # after steps 18 and 19
    _, st_long = gm_ref.solve(csc, db)
    x_full, st_full = gm_ref.solve(csc, db)
    Hfull = gm_ref.hessenberg(K)[:_hcount(K)].copy()
    assert _stats(st_full) == _stats(st_long) == _stats(sts) and np.array_equal(x_full.to_host(), xs)   # repeated solve, same cache
    e1 = np.zeros(K + 1)
    e1[0] = np.linalg.norm(b)
    H = _H_from_raw(Hfull, K)
    rho = [np.linalg.norm(e1[:j + 1] - H[:j + 1, :j] @ np.linalg.lstsq(H[:j + 1, :j], e1[:j + 1], rcond=None)[0]) for j in (18, 19)]
    tol = 0.5 * (rho[0] + rho[1])
    runs = []
    for ce in (None, 1, 3, 8):
        if ce is None:
            opn = _native_csc(nls, ctx, n, csc)
            spy = Spy(_apply_linop(nls, ctx, opn))
            gm = nls.GmresSolver(ctx, n, nls.KrylovJL_GMRES(orth=orth, engine="multikernel", itmax=K), atol=tol, rtol=0.0, keep_hessenberg=_hcount(K))
            try:
                x, st = gm.solve(spy, db)
            finally:
                _lib(nls).b200_linop_destroy(opn)
        else:
            gm = nls.GmresSolver(ctx, n, nls.KrylovJL_GMRES(orth=orth, engine="multikernel", check_every=ce, itmax=K), atol=tol, rtol=0.0, keep_hessenberg=_hcount(K))
            x, st = gm.solve(csc, db)
        runs.append((x.to_host(), _stats(st), gm.hessenberg(st.iters)[:_hcount(st.iters)]))
    assert runs[0][1][:2] == (nls.abi.LS_SOLVED, 19), runs[0][1]
    for x, s, h in runs[1:]:
        assert s == runs[0][1] and np.array_equal(x, runs[0][0]) and np.array_equal(h, runs[0][2]), (regime, orth, s, runs[0][1])
    # a shorter solve after a longer one on the same cache equals the same solve on a fresh cache
    gm = nls.GmresSolver(ctx, n, nls.KrylovJL_GMRES(orth=orth, engine="multikernel", itmax=2 * K), atol=0.0, rtol=0.0, keep_hessenberg=_hcount(2 * K))
    gm.solve(csc, db)
    gm.update_tolerances(atol=tol)
    x2, st2 = gm.solve(csc, db)
    assert _stats(st2) == runs[0][1] and np.array_equal(x2.to_host(), runs[0][0]) and np.array_equal(gm.hessenberg(st2.iters)[:_hcount(st2.iters)], runs[0][2])
    # x0 = 0 passed as a warm start: the same iteration, one more operator application
    gm = nls.GmresSolver(ctx, n, nls.KrylovJL_GMRES(orth=orth, engine="multikernel", warm_start=True, itmax=K), atol=tol, rtol=0.0, keep_hessenberg=_hcount(K))
    xw, stw = gm.solve(csc, db, ctx.zeros(n))
    sw, s0 = _stats(stw), runs[0][1]
    assert (sw[0], sw[1], sw[2], sw[4], sw[5]) == (s0[0], s0[1], s0[2] + 1, s0[4], s0[5]) and np.array_equal(xw.to_host(), runs[0][0])
    assert np.array_equal(gm.hessenberg(stw.iters)[:_hcount(stw.iters)], runs[0][2])


# ----------------------------------------------------------------------------- §5 statuses and preconditioners at G > 1
@pytest.mark.gpu
@pytest.mark.parametrize("orth", ORTHS)
def test_statuses_at_g_above_32(nls, ctx, sizes, orth):
    n = _regime_n(sizes, "G33")
    rng = np.random.default_rng(33)
    # BREAKDOWN: 4 distinct eigenvalues -> the Krylov space is exhausted at k = 4; x is the least-squares (here: exact) solution
    d = np.array([1.0, 3.0, 5.0, 7.0])[np.arange(n) % 4]
    A = sp.diags(d, format="csc")
    b = rng.standard_normal(n) / math.sqrt(n)
    gm = _solver(nls, ctx, n, orth, itmax=20)
    x, st = gm.solve(_csc_device(ctx, A), ctx.to_device(b))
    assert (st.status, st.iters) == (nls.abi.LS_BREAKDOWN, 4), _stats(st)
    assert np.abs(x.to_host() - b / d).max() <= 1e-12 * np.abs(b / d).max()
    # NONFINITE in mid-run: a NaN in the operator's output at step 5 (in the odd tail row of the last CTA): x = x0 bit for bit
    A = _random_sparse(n, seed=3)
    csc = _csc_device(ctx, A)
    op = _native_csc(nls, ctx, n, csc)
    x0 = rng.standard_normal(n)
    try:
        spy = Spy(_apply_linop(nls, ctx, op), nan_at=6, nan_row=n - 1)     # call 1 is A x0 (warm start)
        gm = nls.GmresSolver(ctx, n, nls.KrylovJL_GMRES(orth=orth, engine="multikernel", warm_start=True, itmax=20), atol=0.0, rtol=0.0)
        x, st = gm.solve(spy, ctx.to_device(b), ctx.to_device(x0))
    finally:
        _lib(nls).b200_linop_destroy(op)
    assert (st.status, st.iters) == (nls.abi.LS_NONFINITE, 5) and len(spy.V) == 6, _stats(st)
    assert np.array_equal(x.to_host(), x0)
    # NONFINITE at the start: an Inf in b (tail row)
    bi = b.copy()
    bi[n - 1] = np.inf
    calls = Spy(lambda x, y: None)
    x, st = _solver(nls, ctx, n, orth).solve(calls, ctx.to_device(bi))
    assert (st.status, st.iters, st.nmatvec, len(calls.V)) == (nls.abi.LS_NONFINITE, 0, 0, 0) and not x.to_host().any(), _stats(st)
    # zero right-hand side: solved before any operator application
    x, st = _solver(nls, ctx, n, orth).solve(calls, ctx.zeros(n))
    assert _stats(st) == (nls.abi.LS_SOLVED, 0, 0, 0, 0.0, 0.0, 0.0) and len(calls.V) == 0 and not x.to_host().any()


def _callback_linop(nls, ctx, n, fn):
    def mv(user, x, y):
        try:
            fn(nls.DeviceVector(ctx, n, ptr=y), nls.DeviceVector(ctx, n, ptr=x))
            return 0
        except Exception:  # noqa: BLE001
            import traceback
            traceback.print_exc()
            return 1
    keep = nls.abi.MATVEC_CB(mv)
    op = C.c_void_p()
    _check(nls, ctx, _lib(nls).b200_linop_from_callback(ctx.handle, n, keep, None, C.byref(op)))
    return op, keep


@pytest.mark.gpu
@pytest.mark.parametrize("side", ("left", "right"))
@pytest.mark.parametrize("kind", ("block_jacobi", "multigrid"))
@pytest.mark.parametrize("N", (40, 64))
def test_preconditioned_basis(nls, ctx, po, N, kind, side):
    """The built-in preconditioner wrapped in a spy callback.  Left: the spy operator records v_j and A v_j, the spy
    preconditioner records M^-1 A v_j: Arnoldi relation of M^-1 A.  Right: the spy preconditioner records v_j and N^-1 v_j, the
    spy operator A N^-1 v_j, and the last preconditioner call receives V_k y, whose image must be x (the Pr path of the final
    update).  The same solve with the native preconditioner (status polled every other step) is identical bit for bit."""
    f, P = nls.Brusselator3D(N), po.OracleProblem.bruss3d(N)
    dp = nls._DeviceProblem(ctx, nls.NonlinearProblem(f, None, (3.4, 1.0, 10.0), ctx=ctx))
    u = P.u0(1)
    du = ctx.to_device(u)
    n = P.n
    geo = Geometry(n, ctx.sm_count())
    b = P.residual(u)
    K = 30
    code = {"left": (nls.abi.PRECOND_BLOCK_JACOBI_LEFT, nls.abi.PRECOND_MULTIGRID_LEFT),
            "right": (nls.abi.PRECOND_BLOCK_JACOBI_RIGHT, nls.abi.PRECOND_MULTIGRID_RIGHT)}[side][kind == "multigrid"]

    def native():
        h = C.c_void_p()
        _check(nls, ctx, _lib(nls).b200_linop_precond(dp.handle, du.ptr, code, C.byref(h)))
        return h
    inner = native()
    pspy = Spy(_apply_linop(nls, ctx, inner), keep_out=True)
    pop, keep = _callback_linop(nls, ctx, n, pspy)
    opspy = Spy(lambda x, y: dp.jvp(du, x, out=y), keep_out=True)
    sides = lambda h: {"Pl": h} if side == "left" else {"Pr": h}       # noqa: E731
    gm = nls.GmresSolver(ctx, n, nls.KrylovJL_GMRES(orth="cgs2", engine="multikernel", itmax=K), atol=0.0, rtol=0.0, keep_hessenberg=_hcount(K))
    try:
        x, st = gm.solve(opspy, ctx.to_device(b), **sides(pop))
    finally:
        _lib(nls).b200_linop_destroy(inner)
    label = "%s %s N=%d (%s)" % (kind, side, N, geo.describe(st.iters))
    assert (st.status, st.iters) == (nls.abi.LS_MAXITERS, K), label
    x = x.to_host()
    H = _H_from_raw(gm.hessenberg(K)[:_hcount(K)], K)
    hop = _bruss_hostop(po, P, u)
    if side == "left":
        assert len(opspy.V) == K and len(pspy.V) == K + 1                  # the first preconditioner call takes r0 = b
        assert np.array_equal(pspy.V[0], b)
        for j in range(K):
            assert np.array_equal(pspy.V[j + 1], opspy.Y[j]), (label, j)   # M^-1 is applied to A v_j
        check_operator_images(opspy.V, opspy.Y, hop, label)
        Vb, W, beta = opspy.V, pspy.Y[1:], np.linalg.norm(pspy.Y[0])
        V, orth, ob = check_arnoldi(Vb, W, H, K, 2, n, label, True)
        check_least_squares(V, H, K, beta, x, np.zeros(n), st.rnorm, label)
    else:
        assert len(pspy.V) == K + 1 and len(opspy.V) == K                  # K basis vectors, then V_k y
        for j in range(K):
            assert np.array_equal(opspy.V[j], pspy.Y[j]), (label, j)       # A is applied to N^-1 v_j
        check_operator_images(opspy.V, opspy.Y, hop, label)
        V, orth, ob = check_arnoldi(pspy.V[:K], opspy.Y, H, K, 2, n, label, True)
        y, _ = check_least_squares(V, H, K, np.linalg.norm(b), pspy.V[K], np.zeros(n), st.rnorm, label)
        assert np.array_equal(x, pspy.Y[K])                                  # x = 0 + N^-1 (V_k y)
    # the native preconditioner: no host polling at every step, the same arithmetic
    gm2 = nls.GmresSolver(ctx, n, nls.KrylovJL_GMRES(orth="cgs2", engine="multikernel", itmax=K), atol=0.0, rtol=0.0, keep_hessenberg=_hcount(K))
    x2, st2 = gm2.solve(nls.JacobianOperator(dp, du), ctx.to_device(b), **sides(native()))
    assert _stats(st2) == _stats(st) and np.array_equal(x2.to_host(), x), label
    assert np.array_equal(_H_from_raw(gm2.hessenberg(K)[:_hcount(K)], K), H)


# ----------------------------------------------------------------------------- §6 the operator kernels
def _ld_dot_cols(A, x):
    """Columns of A' x in long double (64-bit significand): |error| <= gamma_m^{ld} sum |a x|, far below the float64 bound."""
    xl = x.astype(np.longdouble)
    return np.array([np.dot(A[:, c].astype(np.longdouble), xl) for c in range(A.shape[1])])


def _assert_sums(got, exact, absum, m, label):
    bound = gamma(m) * absum + float(m) * 2.0 ** -63 * absum + np.finfo(float).tiny
    err = np.abs(got.astype(np.longdouble) - exact).astype(float)
    assert np.all(err <= bound), "%s: entry %d off by %.3e > %.3e" % (label, int(np.argmax(err / bound)), err.max(), bound[np.argmax(err / bound)])
    _ratio("operator_kernels", err, bound)


@pytest.mark.gpu
def test_gemv_every_branch(nls, ctx):
    rng = np.random.default_rng(42)
    L = _lib(nls)
    # trans = 0 (thread per row) with m odd and even; trans = 1 with n > 4096 columns (CTAs take several columns each)
    for (t, m, n) in ((0, 1023, 77), (0, 1024, 77), (0, 5001, 3), (1, 300, 4096 + 1234), (1, 257, 9000)):
        A = rng.standard_normal((m, n))
        x = rng.standard_normal(n if t == 0 else m)
        dA, dx, dy = ctx.to_device(A.ravel(order="F")), ctx.to_device(x), ctx.zeros(m if t == 0 else n)
        _check(nls, ctx, L.b200_gemv(ctx.handle, t, m, n, dA.ptr, m, dx.ptr, dy.ptr))
        M = A if t == 0 else A.T
        exact = _ld_dot_cols(np.ascontiguousarray(M.T), x)
        _assert_sums(dy.to_host(), exact, np.abs(M) @ np.abs(x), M.shape[1], "gemv trans=%d m=%d n=%d" % (t, m, n))
    # the tall branch: m >= 32768, n <= 64 (partials of 16-column groups, G = min(512, ceil(m / 4096)) CTAs; at m = 2 097 153,
    # 16 x 512 partials fill the context's partials buffer); n = 17 and 33 leave a remainder group
    for m in (32768, 32769, 2097153):
        A = np.asfortranarray(rng.standard_normal((m, 64)))
        x = rng.standard_normal(m)
        dA, dx = ctx.to_device(A.ravel(order="F")), ctx.to_device(x)
        exact_all = _ld_dot_cols(A, x)
        abs_all = np.abs(A).T @ np.abs(x)
        for n in (1, 15, 16, 17, 33, 64):
            dy = ctx.to_device(np.full(n, np.nan))
            _check(nls, ctx, L.b200_gemv(ctx.handle, 1, m, n, dA.ptr, m, dx.ptr, dy.ptr))
            _assert_sums(dy.to_host(), exact_all[:n], abs_all[:n], m, "tall gemv' m=%d n=%d (G=%d)" % (m, n, min(512, -(-m // 4096))))
        del dA


@pytest.mark.gpu
@pytest.mark.parametrize("base", (0, 1))
def test_csc_rows_spmv(nls, ctx, base):
    """Empty rows, empty columns, a dense row, duplicate-free random pattern, index bases 0 and 1."""
    rng = np.random.default_rng(base)
    n = 3001
    A = sp.random(n, n, density=0.002, random_state=base, format="lil")
    A[17, :] = rng.standard_normal(n)                           # a dense row
    A = A.tocsc()
    A[:, 5] = 0.0
    A[:, n - 1] = 0.0                                            # empty columns
    A = A.tocsr()
    for r in (0, 2, n - 2, n - 1):                               # empty rows (also the last one)
        A.data[A.indptr[r]:A.indptr[r + 1]] = 0.0
    A.eliminate_zeros()
    A = A.tocsc()
    A.sort_indices()
    assert np.diff(A.tocsr().indptr)[[0, 2, n - 1]].max() == 0 and np.diff(A.indptr)[[5, n - 1]].max() == 0
    csc = _csc_device(ctx, A, base)
    op = _native_csc(nls, ctx, n, csc)
    x = rng.standard_normal(n)
    dy, dx = ctx.to_device(np.full(n, np.nan)), ctx.to_device(x)
    try:
        _check(nls, ctx, _lib(nls).b200_linop_apply(op, dx.ptr, dy.ptr))
    finally:
        _lib(nls).b200_linop_destroy(op)
    Ad = A.toarray()
    exact = _ld_dot_cols(np.ascontiguousarray(Ad.T), x)
    nnz_row = np.diff(A.tocsr().indptr)
    got = dy.to_host()
    assert np.all(got[nnz_row == 0] == 0.0)
    _assert_sums(got, exact, np.abs(Ad) @ np.abs(x), int(nnz_row.max()), "csc spmv base %d" % base)


@pytest.mark.gpu
@pytest.mark.parametrize("dim_N", ((2, 32), (3, 13)))
def test_block_jacobi_kernel(nls, ctx, dim_N):
    """y = D^-1 x with D the 2x2 species blocks on the Brusselator Jacobian's diagonal, against the restated block inverse."""
    dim, N = dim_N
    f = nls.Brusselator2D(N) if dim == 2 else nls.Brusselator3D(N)
    A_, alpha = 3.4, 10.0
    dp = nls._DeviceProblem(ctx, nls.NonlinearProblem(f, None, (A_, 1.0, alpha), ctx=ctx))
    n = dp.n
    NC = n // 2
    rng = np.random.default_rng(N)
    u = rng.uniform(0.1, 3.0, n)
    x = rng.standard_normal(n)
    du = ctx.to_device(u)
    op = C.c_void_p()
    _check(nls, ctx, _lib(nls).b200_linop_block_jacobi(dp.handle, du.ptr, C.byref(op)))
    dy, dx = ctx.zeros(n), ctx.to_device(x)
    try:
        _check(nls, ctx, _lib(nls).b200_linop_apply(op, dx.ptr, dy.ptr))
    finally:
        _lib(nls).b200_linop_destroy(op)
    dx = 1.0 / (N - 1)                                          # the problem's a = alpha / dx^2 (create_bruss)
    a = alpha / (dx * dx)
    lapdiag = -(6.0 if dim == 3 else 4.0) * a
    uc, vc = u[:NC].astype(np.longdouble), u[NC:].astype(np.longdouble)
    d00 = lapdiag + (2 * uc * vc - (A_ + 1)); d01 = uc * uc; d10 = A_ - 2 * uc * vc; d11 = lapdiag - uc * uc
    det = d00 * d11 - d01 * d10
    x0, x1 = x[:NC].astype(np.longdouble), x[NC:].astype(np.longdouble)
    y0, y1 = (d11 * x0 - d01 * x1) / det, (d00 * x1 - d10 * x0) / det
    got = dy.to_host()
    # first-order bound: entries of D (each a sum of <= 3 rounded terms), det, the two products and the quotient
    m00 = abs(lapdiag) + 2 * np.abs(uc * vc) + (A_ + 1); m01 = np.abs(uc * uc); m10 = A_ + 2 * np.abs(uc * vc); m11 = abs(lapdiag) + np.abs(uc * uc)
    mdet = m00 * m11 + m01 * m10
    adet = np.abs(det)
    b0 = gamma(12) * ((m11 * np.abs(x0) + m01 * np.abs(x1)) / adet + np.abs(y0) * mdet / adet)
    b1 = gamma(12) * ((m00 * np.abs(x1) + m10 * np.abs(x0)) / adet + np.abs(y1) * mdet / adet)
    e0 = np.abs(got[:NC] - y0).astype(float)
    e1 = np.abs(got[NC:] - y1).astype(float)
    assert np.all(e0 <= b0.astype(float)) and np.all(e1 <= b1.astype(float)), (e0.max(), e1.max())
    _ratio("block_jacobi", np.concatenate([e0, e1]), np.concatenate([b0, b1]).astype(float))
