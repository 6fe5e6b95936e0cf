"""The resident Arnoldi kernel in every row-geometry regime, and at every split of its rows between the shared-memory stages
and global memory.

`resident3g_arnoldi_kernel` (csrc/gmres.cu, DESIGN §4a) gives CTA b the cells [b*cpc, (b+1)*cpc) of both species; thread `tid`
carries the row pairs 2*(tid + 256*q), q = 0 .. 29, of the CTA's rows (first species' segment, then the second's).  Every basis
vector passes through both kinds of stage:
  * the two shared-memory stages hold the pairs q < qs (TMA copies); the pairs q >= qs are read from global memory ("global tail");
  * the register stage holds the pairs q < 16 in registers and q = 16 .. 29 in a shared-memory "annex" filled by cp.async.
Which of these paths a row takes depends on the rows per CTA and on qs.  `geometry` restates the host-side selection of
`b200_gmres_solve`; the tests use it to choose the smallest grids that reach each regime on the device they run on, to assert
that the regime was reached, and to name the storage class of the rows where a result goes wrong.
B200_RESIDENT_STAGE_PAIRS caps qs, moving rows from the stages to the global tail with the same arithmetic: the results must not
change by a single bit.
"""
import numpy as np
import pytest

R3_THREADS, R3_RP, R3_RPR = 256, 30, 16          # threads per CTA, row pairs per thread, register-held pairs of the register stage
ANNEX_BYTES = (R3_RP - R3_RPR) * R3_THREADS * 16
PAIR = 2 * R3_THREADS                            # rows per q across a CTA
ENV = "B200_RESIDENT_STAGE_PAIRS"
ITMAX = 40
STORAGE = ("stage/register", "stage/annex", "global tail/register", "global tail/annex")


class Geometry:
    """Row map of the resident engine for `n_cells` cells on G CTAs (mirrors the rs_* block of b200_gmres_solve).  Storage
    classes are named `<shared-memory-stage path>/<register-stage path>`: 'stage' or 'global tail', then 'register' or 'annex'."""

    def __init__(self, n_cells, G, smem_optin, qs_cap=None):
        self.n_cells, self.G = n_cells, G
        cpc = -(-n_cells // G)
        self.cpc = cpc + (cpc & 1)
        self.rows_per_cta = 2 * self.cpc
        self.pairs = -(-self.rows_per_cta // PAIR)
        spare = smem_optin - ANNEX_BYTES - 2048 if smem_optin > ANNEX_BYTES + 2048 else 0
        self.qs = min(R3_RP, self.pairs, spare // (2 * 8 * PAIR))
        if qs_cap is not None:
            self.qs = min(self.qs, qs_cap)
        self.stage_words = min(self.rows_per_cta, PAIR * self.qs)
        self.ncell = np.clip(n_cells - self.cpc * np.arange(G), 0, self.cpc)
        self.last_ncell = int(self.ncell[-1])
        self.empty_ctas = int((self.ncell == 0).sum())
        self.srow = np.minimum(2 * self.ncell, PAIR * self.qs)          # rows [0, srow) of each CTA are staged
        self.fits = n_cells % 2 == 0 and G <= 159 and self.rows_per_cta <= 2 * R3_RP * R3_THREADS and self.qs >= 1

    def givens_staged(self, k):
        """Does CTA 0 run the Givens recurrence of Arnoldi step k on a shared-memory copy (the stages, 2 * stage_words doubles)?"""
        return 3 * k <= 2 * self.stage_words

    def row_class(self, row):
        """Global row(s) -> (CTA, thread, q, species, storage index into STORAGE)."""
        row = np.asarray(row, dtype=np.int64)
        s = (row >= self.n_cells).astype(np.int64)
        c = row - s * self.n_cells
        b = c // self.cpc
        lr = s * self.ncell[b] + (c - b * self.cpc)
        p = lr // 2
        q = p // R3_THREADS
        storage = 2 * (q >= self.qs) + (q >= R3_RPR)
        return b, p % R3_THREADS, q, s, storage


def geometry(n_cells, G, smem_optin, qs_cap=None):
    return Geometry(n_cells, G, smem_optin, qs_cap)


def _device(ctx):
    import torch
    return ctx.sm_count(), torch.cuda.get_device_properties(0).shared_memory_per_block_optin


def _cells(dim, N):
    return N ** dim


def _regime_size(dim, G, smem, pairs):
    """Smallest even N whose CTAs carry `pairs` row pairs per thread (at least `pairs` for pairs >= 27), and that fits."""
    for N in range(4, 2000, 2):
        g = geometry(_cells(dim, N), G, smem)
        if g.pairs > R3_RP or not g.fits:
            break
        if g.pairs == pairs or (pairs >= 27 and g.pairs >= pairs):
            return N, g
    pytest.skip("no %dD grid reaches %d row pairs per thread on this device" % (dim, pairs))


def _by_class(g, dev):
    """The worst of a per-row deviation in each row class (species x storage) where it is not zero, worst class first."""
    rows = np.arange(dev.size)
    b, tid, q, s, st = g.row_class(rows)
    key = 4 * s + st
    parts = []
    for k in np.unique(key):
        idx = np.flatnonzero(key == k)
        i = idx[np.argmax(dev[idx])]
        if dev[i] == 0.0:
            continue
        parts.append((dev[i], "species %d %s: %.3g at row %d (CTA %d, thread %d, q %d; %d rows)" % (s[i], STORAGE[st[i]], dev[i], i, b[i], tid[i], q[i], idx.size)))
    parts.sort(key=lambda t: -t[0])
    return "; ".join(p for _, p in parts)


def _column_dev(h, href, iters):
    """Per Hessenberg column: max |h - href| relative to the column's largest entry (columns are stored k + 1 entries each)."""
    out, off = [], 0
    for k in range(1, iters + 1):
        sl = slice(off, off + k + 1)
        off += k + 1
        out.append(np.abs(h[sl] - href[sl]).max() / np.abs(href[sl]).max())
    return np.array(out)


def _setup(nls, ctx, po, dim, N):
    f = nls.Brusselator2D(N) if dim == 2 else nls.Brusselator3D(N)
    P = po.OracleProblem.bruss2d(N) if dim == 2 else po.OracleProblem.bruss3d(N)
    dp = nls._DeviceProblem(ctx, nls.NonlinearProblem(f, None, (3.4, 1.0, 10.0), ctx=ctx))
    u = P.u0(1)
    return P, dp, u, P.residual(u)


# ------------------------------------------------------------------------------------------------ the geometry itself (no GPU)
def test_geometry_matches_the_h100_numbers():
    G, smem = 132, 232448                        # H100 SXM: 132 SMs, 227 KB of opt-in shared memory per block
    g = geometry(100 ** 3, G, smem)
    assert (g.cpc, g.pairs, g.qs, g.last_ncell, g.empty_ctas) == (7576, 30, 21, 7544, 0) and g.fits
    assert int(g.srow[0]) == 21 * PAIR and 21 * PAIR > 7576           # the stages end inside the second species
    assert geometry(80 ** 3, G, smem).pairs == 16
    g = geometry(88 ** 3, G, smem)
    assert (g.pairs, g.qs) == (21, 21) and np.all(g.srow == 2 * g.ncell)  # annex in use, the stages hold every row
    assert geometry(90 ** 3, G, smem).pairs == 22
    assert not geometry(102 ** 3, G, smem).fits and not geometry(1008 ** 2, G, smem).fits
    g = geometry(1006 ** 2, G, smem)
    assert g.fits and g.cpc == 7668
    # small grids leave CTAs empty; the Givens recurrence leaves the stages at k = 342 for 3D N = 48 with one staged pair
    assert geometry(16 ** 3, G, smem).empty_ctas > 0
    g1, gu = geometry(48 ** 3, G, smem, qs_cap=1), geometry(48 ** 3, G, smem)
    assert g1.givens_staged(341) and not g1.givens_staged(342) and gu.givens_staged(400)
    # row map: the first row of CTA 1's second species, and the last row of the grid
    g = geometry(100 ** 3, G, smem)
    assert tuple(map(int, g.row_class(100 ** 3 + 7576))) == (1, 204, 14, 1, 0)     # local row 7576: pair 3788 = 14 * 256 + 204
    assert tuple(map(int, g.row_class(2 * 100 ** 3 - 1))) == (131, 119, 29, 1, 3)  # local row 15087 of the last CTA (7544 cells)


# ------------------------------------------------------------------------------------------------ storage-class probes
@pytest.mark.gpu
@pytest.mark.parametrize("qs_cap", [None, "prefix"])
def test_storage_class_probes(nls, ctx, po, qs_cap, monkeypatch):
    """One storage class at a time.  Through the assembled-operator path with every off-diagonal value set to zero, a
    right-hand side that lives on the rows of one class keeps every basis vector there, so only that class's storage path
    carries data.  The diagonal is drawn from [1, 100]: 8 steps leave the residual far above the level at which MGS loses
    orthogonality, so every Hessenberg entry is reproducible to rounding.  A read from the wrong place shows up in the probe of
    the class whose path is broken: a wrong iterate there, or non-zero rows outside it.  The 22-pair grid uncapped (both
    species staged, a second-species tail) and with the stages capped inside the first species' segment (a first-species tail)."""
    G, smem = _device(ctx)
    N, g = _regime_size(3, G, smem, 22)
    if qs_cap == "prefix":
        cap = g.cpc // PAIR
        monkeypatch.setenv(ENV, str(cap))
        g = geometry(g.n_cells, G, smem, cap)
    P, dp, u, _ = _setup(nls, ctx, po, 3, N)
    sj = nls.SparseJacobian(dp)
    sj.fill(ctx.to_device(u))
    rng = np.random.default_rng(22)
    col = np.repeat(np.arange(P.n), np.diff(sj.colptr))
    diag = sj.rowval - 1 == col
    nzh = np.zeros(sj.nnz)
    nzh[diag] = (1.0 + 99.0 * rng.random(P.n))[col[diag]]
    nz = ctx.to_device(nzh)
    _, _, _, s, st = g.row_class(np.arange(P.n))
    key = 4 * s + st
    keys = list(np.unique(key))
    if qs_cap == "prefix":
        assert 0 * 4 + 2 in keys                                        # first-species rows in the global tail
    else:
        assert 1 * 4 + 0 in keys and 1 * 4 + 3 in keys                  # second-species rows staged, and in the tail (annex)
    full = rng.standard_normal(P.n)
    k_it = 8
    cnt = k_it * (k_it + 3) // 2
    gm = nls.GmresSolver(ctx, P.n, nls.KrylovJL_GMRES(orth="mgs", engine="resident", itmax=k_it), atol=0.0, rtol=0.0, keep_hessenberg=cnt)
    failures = []
    for k in keys:
        rhs = np.where(key == k, full, 0.0)
        xo, so, ho = po.gmres(rhs, csc=(sj.colptr, sj.rowval, nzh, 1), opts=po.default_gmres_opts(atol=0.0, rtol=0.0, orth=po.ORTH_MGS, itmax=k_it), want_hessenberg=cnt)
        x, stt = gm.solve(("sparse_jac", sj, nz), ctx.to_device(rhs))
        x = x.to_host()
        inside = key == k
        xdev = np.abs(x[inside] - xo[inside]).max() / np.abs(xo).max()
        hdev = np.abs(gm.hessenberg(k_it)[:cnt] - ho[:cnt]).max() / np.abs(ho[:cnt]).max()
        leak = np.where(inside, 0.0, np.abs(x) / np.abs(xo).max())
        if not (stt.iters == so.iters == k_it and hdev <= 1e-10 and xdev <= 1e-10 and leak.max() == 0.0):
            failures.append("probe of species %d %s: iters %d, Hessenberg %.3g, iterate %.3g%s" % (
                k // 4, STORAGE[k % 4], stt.iters, hdev, xdev, "; rows outside it not zero: " + _by_class(g, leak) if leak.max() > 0.0 else ""))
    assert not failures, "N %d, qs %d: %s" % (N, g.qs, " | ".join(failures))


# ------------------------------------------------------------------------------------------------ a. regime sweep vs the oracle
def _oracle_with_sensitivity(po, b, cnt, resid, **kw):
    """The oracle's GMRES, its reproducibility under a reordering of its sums (1 thread vs all threads: the envelope the
    Arnoldi recurrence leaves for another implementation), and the gap between its residual estimate and its true residual."""
    nthreads = po.get_threads()
    xo, so, ho = po.gmres(b, want_hessenberg=cnt, **kw)
    po.set_threads(1)
    try:
        x1, s1, h1 = po.gmres(b, want_hessenberg=cnt, **kw)
    finally:
        po.set_threads(nthreads)
    env = np.maximum.accumulate(_column_dev(h1, ho, ITMAX))
    xenv = np.abs(x1 - xo).max() / np.abs(xo).max()
    gap = max(abs(np.linalg.norm(resid(xo)) - so.rnorm), abs(np.linalg.norm(resid(x1)) - s1.rnorm))
    return xo, so, ho, env, xenv, gap


def _check_against_oracle(g, b, x, st, hg, xo, so, ho, env, xenv, gap, resid):
    ro, rg = resid(xo), resid(x)
    where = "%s | x: %s | b - J x: %s" % (
        "cpc %d, pairs %d, qs %d" % (g.cpc, g.pairs, g.qs),
        _by_class(g, np.abs(x - xo) / np.abs(xo).max()), _by_class(g, np.abs(rg - ro) / np.abs(b).max()))
    assert st.iters == so.iters == ITMAX, where
    dev = _column_dev(hg, ho, ITMAX)
    assert dev[:10].max() <= 1e-10, "Hessenberg columns 1-10 %s; %s" % (dev[:10], where)
    # the oracle's all-thread run is itself one draw from that reordering (OpenMP reductions), hence the wide factor
    bound = 100.0 * env + 1e-11
    assert np.all(dev <= bound) and dev.max() <= 5e-6, "Hessenberg %.3g of its bound, max %.3g; %s" % ((dev / bound).max(), dev.max(), where)
    assert abs(st.rnorm0 - so.rnorm0) <= 1e-12 * so.rnorm0, where
    assert np.abs(x - xo).max() <= max(30.0 * xenv, 1e-9) * np.abs(xo).max(), where
    # the Givens estimate tracks the true residual as closely as the oracle's does: a wrong row in any basis vector breaks
    # the Arnoldi relation A V_k = V_{k+1} H_k that the estimate rests on, even where H itself looks plausible
    tgap = abs(np.linalg.norm(rg) - st.rnorm)
    assert tgap <= max(30.0 * gap, 1e-13 * so.rnorm0), "true-residual gap %.3g (oracle %.3g); %s" % (tgap, gap, where)


REGIMES = [16, 17, 21, 22, 27]


@pytest.mark.gpu
@pytest.mark.parametrize("orth", ["mgs", "cgs2"])
@pytest.mark.parametrize("dim", [3, 2])
@pytest.mark.parametrize("pairs", REGIMES)
def test_regime_matrix_free_vs_oracle(nls, ctx, po, pairs, dim, orth):
    G, smem = _device(ctx)
    N, g = _regime_size(dim, G, smem, pairs)
    if dim == 3 and N == 100:
        pytest.skip("3D N = 100 is covered by test_gpu_n100_parity.py")
    assert g.pairs == pairs or (pairs >= 27 and g.pairs >= 27), (N, g.pairs)
    assert (g.pairs > R3_RPR) == (pairs > 16), (N, g.pairs)             # the annex is in use from 17 pairs on
    assert (g.qs < g.pairs) == (pairs >= 22), (N, g.pairs, g.qs)       # and a global tail from 22 on (227 KB of shared memory)
    P, dp, u, b = _setup(nls, ctx, po, dim, N)
    ocode = po.ORTH_MGS if orth == "mgs" else po.ORTH_CGS2
    cnt = ITMAX * (ITMAX + 3) // 2
    resid = lambda x: b - P.jvp(u, x)  # noqa: E731
    ref = _oracle_with_sensitivity(po, b, cnt, resid, prob=P, u=u, opts=po.default_gmres_opts(atol=1e-8, rtol=3e-13, orth=ocode, itmax=ITMAX))
    gm = nls.GmresSolver(ctx, P.n, nls.KrylovJL_GMRES(orth=orth, engine="resident", itmax=ITMAX), atol=1e-8, rtol=3e-13, keep_hessenberg=cnt)
    x, st = gm.solve(nls.JacobianOperator(dp, ctx.to_device(u)), ctx.to_device(b))
    _check_against_oracle(g, b, x.to_host(), st, gm.hessenberg(st.iters)[:cnt], *ref, resid)


@pytest.mark.gpu
@pytest.mark.parametrize("dim,pairs,orth", [(3, 17, "mgs"), (2, 21, "cgs2"), (3, 22, "mgs")])
def test_regime_assembled_sparse_vs_oracle(nls, ctx, po, dim, pairs, orth):
    G, smem = _device(ctx)
    N, g = _regime_size(dim, G, smem, pairs)
    P, dp, u, b = _setup(nls, ctx, po, dim, N)
    sj = nls.SparseJacobian(dp)
    nz = sj.fill(ctx.to_device(u))
    nzh = nz.to_host()
    ocode = po.ORTH_MGS if orth == "mgs" else po.ORTH_CGS2
    cnt = ITMAX * (ITMAX + 3) // 2
    resid = lambda x: b - po.spmv(P.n, sj.colptr, sj.rowval, nzh, x)  # noqa: E731
    ref = _oracle_with_sensitivity(po, b, cnt, resid, csc=(sj.colptr, sj.rowval, nzh, 1), opts=po.default_gmres_opts(atol=1e-8, rtol=3e-13, orth=ocode, itmax=ITMAX))
    gm = nls.GmresSolver(ctx, P.n, nls.KrylovJL_GMRES(orth=orth, engine="resident", itmax=ITMAX), atol=1e-8, rtol=3e-13, keep_hessenberg=cnt)
    x, st = gm.solve(("sparse_jac", sj, nz), ctx.to_device(b))
    _check_against_oracle(g, b, x.to_host(), st, gm.hessenberg(st.iters)[:cnt], *ref, resid)


# ------------------------------------------------------------------------------------------------ b. stage-split invariance
def _run(nls, ctx, n, A, b, orth, itmax, rtol=3e-13, atol=1e-8):
    cnt = itmax * (itmax + 3) // 2
    gm = nls.GmresSolver(ctx, n, nls.KrylovJL_GMRES(orth=orth, engine="resident", itmax=itmax), atol=atol, rtol=rtol, keep_hessenberg=cnt)
    x, st = gm.solve(A, b)
    return st.iters, st.rnorm, gm.hessenberg(st.iters), x.to_host()


def _assert_same(ref, got, what):
    assert ref[0] == got[0], (what, ref[0], got[0])
    assert ref[1] == got[1], (what, ref[1], got[1])
    assert np.array_equal(ref[2], got[2]), (what, "Hessenberg", np.flatnonzero(ref[2] != got[2])[:5])
    assert np.array_equal(ref[3], got[3]), (what, "x", np.abs(ref[3] - got[3]).max())


def _caps(g):
    """1, the largest cap whose stages end inside the first species' segment (the species-0-only prefix), one more, and the
    uncapped number of staged pairs."""
    f = g.cpc // PAIR
    return sorted({c for c in (1, f, f + 1, g.qs) if 1 <= c <= g.qs})


@pytest.mark.gpu
def test_stage_pairs_variable_is_read(nls, ctx, po, monkeypatch):
    P, dp, u, b = _setup(nls, ctx, po, 3, 16)
    for bad in ("0", str(R3_RP + 1), "x"):
        monkeypatch.setenv(ENV, bad)
        gm = nls.GmresSolver(ctx, P.n, nls.KrylovJL_GMRES(engine="resident", itmax=4), atol=0.0, rtol=1e-10)
        with pytest.raises(nls.abi.B200Error) as e:
            gm.solve(nls.JacobianOperator(dp, ctx.to_device(u)), ctx.to_device(b))
        assert e.value.code == nls.abi.ERR_INVALID and ENV in str(e.value), bad
    monkeypatch.setenv(ENV, str(R3_RP))                                 # the largest value is accepted (and changes nothing)
    gm = nls.GmresSolver(ctx, P.n, nls.KrylovJL_GMRES(engine="resident", itmax=4), atol=0.0, rtol=1e-10)
    gm.solve(nls.JacobianOperator(dp, ctx.to_device(u)), ctx.to_device(b))


@pytest.mark.gpu
@pytest.mark.parametrize("orth", ["mgs", "cgs2"])
@pytest.mark.parametrize("N,csr", [(16, False), (64, False), ("22 pairs", False), (100, False), (100, True)])
def test_stage_split_is_bit_identical(nls, ctx, po, monkeypatch, N, csr, orth):
    G, smem = _device(ctx)
    if N == "22 pairs":
        N, _ = _regime_size(3, G, smem, 22)
    g = geometry(N ** 3, G, smem)
    assert g.fits
    f = g.cpc // PAIR
    if 1 <= f < g.qs:                     # the cap f leaves the stages inside the first species' segment of a full CTA
        assert geometry(N ** 3, G, smem, f).srow[0] <= g.cpc
    P, dp, u, b = _setup(nls, ctx, po, 3, N)
    if csr:
        sj = nls.SparseJacobian(dp)
        A = ("sparse_jac", sj, sj.fill(ctx.to_device(u)))
    else:
        A = nls.JacobianOperator(dp, ctx.to_device(u))
    db = ctx.to_device(b)
    monkeypatch.delenv(ENV, raising=False)
    ref = _run(nls, ctx, P.n, A, db, orth, ITMAX)
    for cap in _caps(g):
        monkeypatch.setenv(ENV, str(cap))
        _assert_same(ref, _run(nls, ctx, P.n, A, db, orth, ITMAX), "N %d cap %d (qs %d)" % (N, cap, g.qs))


def _boundary_sizes(G, smem):
    """2D grids on which the stages end exactly at a CTA's species boundary (srow == ncell) for some cap: the smallest and the
    largest with every full CTA so, and the smallest with only the last CTA so."""
    full, last = [], []
    for N in range(4, 2000, 2):
        g = geometry(N * N, G, smem)
        if not g.fits:
            break
        if g.cpc % PAIR == 0 and g.cpc // PAIR <= g.qs:
            full.append((N, g.cpc // PAIR))
        elif g.last_ncell > 0 and g.last_ncell % PAIR == 0 and g.last_ncell // PAIR <= g.qs:
            last.append((N, g.last_ncell // PAIR))
    return sorted(set(full[:1] + full[-1:] + last[:1]))


@pytest.mark.gpu
def test_stages_ending_at_the_species_boundary_are_bit_identical(nls, ctx, po, monkeypatch):
    G, smem = _device(ctx)
    sizes = _boundary_sizes(G, smem)
    assert sizes
    for N, cap in sizes:
        g = geometry(N * N, G, smem, cap)
        assert np.any((g.srow == g.ncell) & (g.ncell > 0)), (N, cap)
        P, dp, u, b = _setup(nls, ctx, po, 2, N)
        A, db = nls.JacobianOperator(dp, ctx.to_device(u)), ctx.to_device(b)
        monkeypatch.delenv(ENV, raising=False)
        ref = _run(nls, ctx, P.n, A, db, "mgs", ITMAX)
        monkeypatch.setenv(ENV, str(cap))
        _assert_same(ref, _run(nls, ctx, P.n, A, db, "mgs", ITMAX), "2D N %d cap %d" % (N, cap))


@pytest.mark.gpu
def test_unstaged_givens_tail_is_bit_identical(nls, ctx, po, monkeypatch):
    """With one staged pair at 3D N = 48 the Givens recurrence of CTA 0 no longer fits the stages from k = 342 on and runs on
    global memory; uncapped it stays staged for all 400 steps."""
    N, itmax = 48, 400
    G, smem = _device(ctx)
    g1, gu = geometry(N ** 3, G, smem, 1), geometry(N ** 3, G, smem)
    k0 = next(k for k in range(1, itmax + 1) if not g1.givens_staged(k))
    assert k0 < itmax and gu.givens_staged(itmax), (k0, gu.stage_words)
    P, dp, u, b = _setup(nls, ctx, po, 3, N)
    A, db = nls.JacobianOperator(dp, ctx.to_device(u)), ctx.to_device(b)
    monkeypatch.delenv(ENV, raising=False)
    ref = _run(nls, ctx, P.n, A, db, "mgs", itmax, rtol=1e-14, atol=0.0)
    assert ref[0] > k0, (ref[0], k0)
    monkeypatch.setenv(ENV, "1")
    _assert_same(ref, _run(nls, ctx, P.n, A, db, "mgs", itmax, rtol=1e-14, atol=0.0), "3D N 48 cap 1")


# ------------------------------------------------------------------------------------------------ c. capacity boundary
def _largest_fitting_2d(G, smem):
    best = None
    for N in range(4, 2000, 2):
        if geometry(N * N, G, smem).fits:
            best = N
        elif best is not None and geometry(N * N, G, smem).rows_per_cta > 2 * R3_RP * R3_THREADS:
            return best, N
    pytest.skip("no 2D grid exceeds the resident engine's capacity")


@pytest.mark.gpu
def test_capacity_boundary(nls, ctx, po):
    G, smem = _device(ctx)
    N, N_over = _largest_fitting_2d(G, smem)
    g = geometry(N * N, G, smem)
    assert g.pairs == R3_RP and g.rows_per_cta > 2 * (R3_RP - 1) * R3_THREADS
    P, dp, u, b = _setup(nls, ctx, po, 2, N)
    k = 10
    cnt = k * (k + 3) // 2
    xo, so, ho = po.gmres(b, prob=P, u=u, opts=po.default_gmres_opts(atol=1e-8, rtol=3e-13, orth=po.ORTH_MGS, itmax=k), want_hessenberg=cnt)
    gm = nls.GmresSolver(ctx, P.n, nls.KrylovJL_GMRES(orth="mgs", engine="resident", itmax=k), atol=1e-8, rtol=3e-13, keep_hessenberg=cnt)
    x, st = gm.solve(nls.JacobianOperator(dp, ctx.to_device(u)), ctx.to_device(b))
    assert st.iters == so.iters == k
    dev = _column_dev(gm.hessenberg(k)[:cnt], ho[:cnt], k)
    assert dev.max() <= 1e-10, (N, dev)
    # one step past the capacity, in 2D and 3D: the explicit request refuses, automatic selection takes the multi-kernel engine
    N3 = next(n for n in range(4, 200, 2) if not geometry(n ** 3, G, smem).fits and geometry(n ** 3, G, smem).rows_per_cta > 2 * R3_RP * R3_THREADS)
    for dim, n_ in ((2, N_over), (3, N3)):
        P, dp, u, b = _setup(nls, ctx, po, dim, n_)
        A, db = nls.JacobianOperator(dp, ctx.to_device(u)), ctx.to_device(b)
        gm = nls.GmresSolver(ctx, P.n, nls.KrylovJL_GMRES(engine="resident", itmax=k), atol=0.0, rtol=1e-10)
        with pytest.raises(nls.abi.B200Error) as e:
            gm.solve(A, db)
        assert e.value.code == nls.abi.ERR_UNSUPPORTED, (dim, n_)
        xa, sa = nls.GmresSolver(ctx, P.n, nls.KrylovJL_GMRES(engine="auto", itmax=k), atol=0.0, rtol=1e-10).solve(A, db)
        xm, sm = nls.GmresSolver(ctx, P.n, nls.KrylovJL_GMRES(engine="multikernel", itmax=k), atol=0.0, rtol=1e-10).solve(A, db)
        assert sa.iters == sm.iters == k and sa.rnorm < sa.rnorm0 and np.array_equal(xa.to_host(), xm.to_host()), (dim, n_)
