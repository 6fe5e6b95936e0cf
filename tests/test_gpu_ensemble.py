"""The batched ensemble kernel (`ens_newton_kernel`, csrc/ens_batched.cu; BASELINE config 5) in every row-walk geometry,
queue depth and option set, against three references:

* the per-trajectory C oracle (`po.ensemble_solve` / `OracleProblem.newton`) for the option sets it implements (the three
  AbsNorm modes on the inf-norm, MGS / CGS2, EW forcing, itmax, GMRES atol / rtol, maxiters);
* `residual_ld` below, an independent NumPy restatement of the 2D Brusselator residual (forcing disc, dx = 1/(N-1))
  evaluated in extended precision for every returned iterate;
* the single-system CUDA driver (`nls.solve` on one trajectory, same options) for the option sets the kernel does not
  implement, which `b200_ens_solve` must route to that driver.

Retcodes and `nsteps` match exactly, roots to RTOL_ROOT, `njvp` to +-2 Arnoldi steps per Newton step (reduction order
differs between the kernel and the oracle).

A thread's rows are r = tid + 256 q (q < 8); the kernel walks (species, i, j) from one row to the next by adding
(256 mod N, 256 div N) with carries.  GEOMETRY_N picks sizes where that walk does each thing it can do: nothing (one row
per thread: 3, 9, 11), no i-carry (16, 32), a step of j by N or more, into the second species (12, 13, 15), i-carries
over several steps (17, 22, 23), a partly filled last q (31), and the size just past the kernel's limit that takes the
driver (33)."""
import numpy as np
import pytest

ET, NPT = 256, 8          # threads per CTA and rows per thread of ens_newton_kernel
ALPHA = 10.0
RTOL_ROOT = 1e-6
U_ROUND = 2.0 ** -53
GEOMETRY_N = (3, 9, 11, 12, 13, 15, 16, 17, 22, 23, 31, 32, 33)


# ----------------------------------------------------------------------------- row walk (no GPU)
def walk_rows(N, tid):
    """ENS_ROW_WALK_BEGIN / ENS_ROW_WALK_STEP restated: the (s, i, j) the kernel assigns to rows tid + ET q, q < NPT."""
    NC = N * N
    di, dj = ET % N, ET // N
    s = int(tid >= NC)
    c = tid - s * NC
    j = c // N
    i = c - j * N
    while j >= N:
        j -= N
        s += 1
    out = []
    for q in range(NPT):
        if q > 0:
            i += di
            j += dj
            if i >= N:
                i -= N
                j += 1
            while j >= N:
                j -= N
                s += 1
        out.append((s, i, j))
    return out


def geometry(N):
    n = 2 * N * N
    nq = -(-n // ET)
    return dict(walk_di=ET % N, walk_dj=ET // N, n=n, nq=nq, last_rows=n - ET * (nq - 1))


def test_row_walk_restatement_equals_divmod():
    for N in range(3, 33):
        NC, n = N * N, 2 * N * N
        for tid in range(ET):
            rows = walk_rows(N, tid)
            for q, (s, i, j) in enumerate(rows):
                r = tid + ET * q
                if r < n:
                    assert (s, i, j) == (r // NC, (r % NC) % N, (r % NC) // N), (N, tid, q)
                    # a step into a row the kernel uses crosses at most one species boundary: the carry loop of
                    # ENS_ROW_WALK_STEP runs more than once only on rows past n, which are never evaluated
                    if q > 0:
                        assert s - rows[q - 1][0] <= 1, (N, tid, q)


@pytest.mark.parametrize("N", GEOMETRY_N)
def test_row_walk_regime(N):
    g = geometry(N)
    print("N=%d walk_di=%d walk_dj=%d rows in last q=%d (q < %d)" % (N, g["walk_di"], g["walk_dj"], g["last_rows"], g["nq"]))
    if N > 32:
        assert g["n"] > ET * NPT                       # the kernel refuses it: the driver runs every trajectory
    elif N in (3, 9, 11):
        assert g["nq"] == 1                            # one row per thread, the walk never steps
    elif N in (12, 13, 15):
        assert g["walk_dj"] >= N and g["nq"] >= 2      # every step wraps j past N into the second species
        assert g["walk_di"] > 0
    elif N in (16, 32):
        assert g["walk_di"] == 0                       # the i-carry never runs
    elif N in (17, 22, 23):
        assert 0 < g["walk_di"] and g["walk_dj"] < N and g["nq"] >= 3
    elif N == 31:
        assert g["walk_di"] > 0 and g["nq"] == NPT and g["last_rows"] < ET


# ----------------------------------------------------------------------------- references
def forcing_disc(N):
    """F[j, i] = 5 inside the disc (x_i - 0.3)^2 + (y_j - 0.6)^2 <= 0.1^2, x_i = i / (N - 1) (sparsity_tests__item1.jl:7-12)."""
    x = np.arange(N) / (N - 1)
    return np.where((x[None, :] - 0.3) ** 2 + (x[:, None] - 0.6) ** 2 <= 0.1 ** 2, 5.0, 0.0)


def residual_ld(N, U, A, B, alpha=ALPHA):
    """||f(u_m)||_inf of the 2D Brusselator for every row of U (K, 2 N^2), evaluated in long double, and a bound on how far
    any float64 evaluation of the same formula can be from it: 16 u sum_r |terms of row r| (about ten roundings per row)."""
    K = U.shape[0]
    dx = 1.0 / (N - 1)
    a = np.longdouble(alpha / (dx * dx))
    F = forcing_disc(N).astype(np.longdouble)
    finf, bound = np.empty(K), np.empty(K)
    for lo in range(0, K, 256):
        W = U[lo:lo + 256].reshape(-1, 2, N, N).astype(np.longdouble)  # [k, species, j, i]: vec index = s N^2 + i + N j
        u, v = W[:, 0], W[:, 1]
        Am = np.asarray(A[lo:lo + 256], dtype=np.longdouble)[:, None, None]
        Bm = np.asarray(B[lo:lo + 256], dtype=np.longdouble)[:, None, None]

        def lap(w):
            return np.roll(w, 1, 2) + np.roll(w, -1, 2) + np.roll(w, -1, 1) + np.roll(w, 1, 1) - 4 * w

        def alap(w):
            w = np.abs(w)
            return np.roll(w, 1, 2) + np.roll(w, -1, 2) + np.roll(w, -1, 1) + np.roll(w, 1, 1) + 4 * w

        uuv = u * u * v
        fu = a * lap(u) + Bm + uuv - (Am + 1) * u + F
        fv = a * lap(v) + Am * u - uuv
        su = a * alap(u) + np.abs(Bm) + np.abs(uuv) + np.abs((Am + 1) * u) + F
        sv = a * alap(v) + np.abs(Am * u) + np.abs(uuv)
        fmax = np.maximum(np.abs(fu).max(axis=(1, 2)), np.abs(fv).max(axis=(1, 2)))
        smax = np.maximum(su.max(axis=(1, 2)), sv.max(axis=(1, 2)))
        finf[lo:lo + 256] = fmax.astype(np.float64)
        bound[lo:lo + 256] = (16 * U_ROUND * smax).astype(np.float64)
    return finf, bound


def assert_residuals_consistent(nls, N, out, A, B, abstol):
    """The reported resid_inf[m] is the residual of the returned u[m] (to rounding), for every trajectory; Success means
    it is <= abstol."""
    finf, bound = residual_ld(N, out["u"], A, B)
    resid = out["resid"]
    both_nonfinite = ~np.isfinite(resid) & ~np.isfinite(finf)
    ok = (np.abs(resid - finf) <= bound) | both_nonfinite
    bad = np.flatnonzero(~ok)
    assert bad.size == 0, [(int(m), resid[m], finf[m], bound[m], int(out["rc"][m])) for m in bad[:8]]
    succ = out["rc"] == nls.ReturnCode.Success
    assert np.all(resid[succ] <= abstol) and np.all(finf[succ] <= abstol + bound[succ])
    return finf


def ens_solve(nls, ctx, N, u0, A, B, alg, **kw):
    K = len(A)
    cache = nls.EnsembleCache(ctx, N, K, ALPHA, alg, **kw)
    l0 = ctx.kernel_launches()
    res = cache.solve(ctx.to_device(np.ascontiguousarray(u0, dtype=np.float64).ravel()), ctx.to_device(np.ascontiguousarray(A, dtype=np.float64)),
                      ctx.to_device(np.ascontiguousarray(B, dtype=np.float64)))
    return dict(u=cache.u_out.to_host().reshape(K, -1), resid=cache.resid.to_host(), rc=cache.rc.to_host(), ns=cache.ns.to_host(),
                nj=cache.nj.to_host(), summary=res, launches=ctx.kernel_launches() - l0, cache=cache, u0=u0, A=A, B=B)


def resolve(nls, ctx, out):
    """A second solve on the same cache and inputs."""
    c = out["cache"]
    c.solve(ctx.to_device(np.ascontiguousarray(out["u0"]).ravel()), ctx.to_device(np.ascontiguousarray(out["A"])), ctx.to_device(np.ascontiguousarray(out["B"])))
    return dict(u=c.u_out.to_host().reshape(c.K, -1), resid=c.resid.to_host(), rc=c.rc.to_host(), ns=c.ns.to_host(), nj=c.nj.to_host())


def assert_bit_identical(a, b, rows_a=slice(None), rows_b=slice(None)):
    for key in ("u", "resid", "rc", "ns", "nj"):
        x, y = a[key][rows_a], b[key][rows_b]
        assert np.array_equal(x, y, equal_nan=np.issubdtype(x.dtype, np.floating)), key


def assert_matches_oracle(out, ref, rows=slice(None)):
    uo, ro, rco, nso, njo, _ = ref
    rc, ns, nj, u = out["rc"][rows], out["ns"][rows], out["nj"][rows], out["u"][rows]
    assert np.array_equal(rc, rco), (rc, rco)
    assert np.array_equal(ns, nso), (ns, nso)
    scale = np.maximum(np.abs(uo).max(axis=1), 1e-300)
    err = np.abs(u - uo).max(axis=1) / scale
    assert np.all(err <= RTOL_ROOT), err.max()
    assert np.all(np.abs(nj - njo) <= 2 * nso), np.abs(nj - njo).max()


def oracle(po, N, u0, A, B, **opts):
    return po.ensemble_solve(N, u0, A, B, opts=po.default_newton_opts(**opts))


def start(po, N, K, spread=0.01):
    return np.tile(po.OracleProblem.bruss2d(N).u0(), (K, 1)) * (1.0 + spread * np.arange(K))[:, None]


ORTH = {"mgs": 0, "cgs2": 2}  # po.ORTH_MGS / po.ORTH_CGS2


# ----------------------------------------------------------------------------- 1. row-walk geometry
@pytest.mark.gpu
@pytest.mark.parametrize("N", GEOMETRY_N)
def test_geometry_vs_oracle(nls, ctx, po, N):
    import bench
    K = 6
    A, B = bench.ensemble_params(K)
    u0 = start(po, N, K, 0.03)  # no iterate of these starts has ||f||_inf within 4% of abstol: no ties to break by rounding
    out = ens_solve(nls, ctx, N, u0, A, B, nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(orth="mgs")), abstol=1e-8)
    ref = oracle(po, N, u0, A, B, abstol=1e-8, gmres_orth=po.ORTH_MGS)
    assert np.all(out["rc"] == nls.ReturnCode.Success)
    assert_matches_oracle(out, ref)
    assert_residuals_consistent(nls, N, out, A, B, 1e-8)
    g = geometry(N)
    print("N=%d walk_di=%d walk_dj=%d last q rows=%d launches=%d" % (N, g["walk_di"], g["walk_dj"], g["last_rows"], out["launches"]))
    if N <= 32:
        assert out["launches"] <= 2          # one kernel for the whole batch
    else:
        assert out["launches"] >= 10 * K     # the general driver, trajectory by trajectory


# ----------------------------------------------------------------------------- 2. queue depth and independence
@pytest.mark.gpu
@pytest.mark.parametrize("depth", ["one", "below_sm_count", "above_any_grid"])
def test_queue_depth(nls, ctx, po, depth):
    import bench
    N = 16
    sm = ctx.sm_count()
    K = {"one": 1, "below_sm_count": sm // 2 + 1, "above_any_grid": 8 * sm + 37}[depth]  # 2048 threads per SM / 256 = 8 CTAs at most
    A, B = bench.ensemble_params(K)
    u0 = np.tile(po.OracleProblem.bruss2d(N).u0(), (K, 1)) * (1.0 + 1e-3 * (np.arange(K) % 97))[:, None]
    alg = nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(orth="mgs"))
    out = ens_solve(nls, ctx, N, u0, A, B, alg, abstol=1e-8)
    print("queue depth %s: K=%d, sm_count=%d" % (depth, K, sm))
    assert np.all(out["rc"] == nls.ReturnCode.Success)
    assert_residuals_consistent(nls, N, out, A, B, 1e-8)
    sample = np.unique(np.linspace(0, K - 1, min(K, 48)).astype(int))
    assert_matches_oracle(out, oracle(po, N, u0[sample], A[sample], B[sample], abstol=1e-8, gmres_orth=po.ORTH_MGS), sample)
    for m in sample[:: max(1, len(sample) // 4)]:   # alone in a batch of one: the same bits
        alone = ens_solve(nls, ctx, N, u0[m:m + 1], A[m:m + 1], B[m:m + 1], alg, abstol=1e-8)
        assert_bit_identical(out, alone, slice(m, m + 1))


@pytest.mark.gpu
def test_benchmark_batch_8192_is_exact_and_independent(nls, ctx, po):
    """bench.py's ensemble leg (K = 8192, 2D N = 32, MGS, abstol 1e-8): every trajectory converges to a true root, and a
    trajectory's bits depend neither on the CTA that ran it nor on what ran before it."""
    import bench
    N, K = 32, 8192
    A, B = bench.ensemble_params(K)
    dp = nls._DeviceProblem(ctx, nls.NonlinearProblem(nls.Brusselator2D(N), None, (3.4, 1.0, ALPHA), ctx=ctx))
    u0 = np.tile(dp.u0().to_host(), (K, 1))
    alg = nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(orth="mgs"))
    out = ens_solve(nls, ctx, N, u0, A, B, alg, abstol=1e-8)
    assert out["summary"].nsuccess == K and np.all(out["rc"] == nls.ReturnCode.Success)
    finf = assert_residuals_consistent(nls, N, out, A, B, 1e-8)
    assert finf.max() < 1e-8
    # a 64-trajectory sample spread over the (A, B) grid, solved as its own batch
    sample = np.unique(np.concatenate([[0, 63, 64, 127, 4095, 4096, 8128, 8191], np.linspace(1, 8190, 56).astype(int)]))
    alone = ens_solve(nls, ctx, N, u0[sample], A[sample], B[sample], alg, abstol=1e-8)
    assert_bit_identical(out, alone, sample)
    # a permuted batch gives the permuted results
    perm = np.random.default_rng(8192).permutation(K)
    permuted = ens_solve(nls, ctx, N, u0[perm], A[perm], B[perm], alg, abstol=1e-8)
    assert_bit_identical(out, permuted, perm)
    # a second solve on the same cache
    assert_bit_identical(out, resolve(nls, ctx, out))
    # 16 of the sample against the oracle
    s16 = sample[:: len(sample) // 16][:16]
    assert_matches_oracle(out, oracle(po, N, u0[s16], A[s16], B[s16], abstol=1e-8, gmres_orth=po.ORTH_MGS), s16)


# ----------------------------------------------------------------------------- 3. partial deferral
@pytest.mark.gpu
def test_partial_deferral_is_exact(nls, ctx, po, monkeypatch):
    """With the basis slab between the trajectories' Krylov needs, each trajectory is either solved in the kernel (the same
    bits as with the default 512 columns) or redone by the general driver (the same bits as the driver alone)."""
    import bench
    N, K = 16, 12
    A, B = bench.ensemble_params(K)
    u0 = start(po, N, K, 0.25)
    need = []
    for m in range(K):  # the most Arnoldi steps any Newton step of trajectory m takes
        _, _, _, tr = po.OracleProblem.bruss2d(N, A=A[m], B=B[m]).newton(u0[m], po.default_newton_opts(abstol=1e-8, gmres_orth=po.ORTH_MGS))
        need.append(max(t.lin_iters for t in tr))
    need = np.array(need)
    cap = 94
    assert need.min() <= cap - 2 and need.max() >= cap + 3, need   # both kinds, with room for +-2 steps of reduction order
    alg = nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(orth="mgs"))
    r512 = ens_solve(nls, ctx, N, u0, A, B, alg, abstol=1e-8)
    rdrv = dict(u=np.empty_like(r512["u"]), resid=np.empty(K), rc=np.empty(K, np.int32), ns=np.empty(K, np.int32), nj=np.empty(K, np.int32))
    for m in range(K):
        sol = nls.solve(nls.NonlinearProblem(nls.Brusselator2D(N), u0[m].copy(), (A[m], B[m], ALPHA), ctx=ctx), alg, abstol=1e-8, store_trace=False)
        rdrv["u"][m], rdrv["resid"][m], rdrv["rc"][m], rdrv["ns"][m], rdrv["nj"][m] = sol.u, sol.resid_inf, sol.retcode, sol.stats.nsteps, sol.stats.njvp
    monkeypatch.setenv("B200_ENS_BASIS_COLUMNS", str(cap))
    rmid = ens_solve(nls, ctx, N, u0, A, B, alg, abstol=1e-8)
    monkeypatch.setenv("B200_ENS_BASIS_COLUMNS", "2")
    rall = ens_solve(nls, ctx, N, u0, A, B, alg, abstol=1e-8)
    monkeypatch.delenv("B200_ENS_BASIS_COLUMNS")

    def same(a, b, m):
        return all(np.array_equal(a[k][m], b[k][m]) for k in ("u", "resid", "rc", "ns", "nj"))

    as512 = np.array([same(rmid, r512, m) for m in range(K)])
    asdrv = np.array([same(rmid, rdrv, m) for m in range(K)])
    print("cap %d: oracle needs %s; %d trajectories deferred" % (cap, need.tolist(), int((asdrv & ~as512).sum())))
    assert np.all(as512 | asdrv), (as512, asdrv)
    assert np.any(as512 & ~asdrv) and np.any(asdrv & ~as512)
    assert np.array_equal(asdrv & ~as512, need > cap)
    assert all(same(rall, rdrv, m) for m in range(K))                 # cap 2: every trajectory deferred
    assert np.all(r512["rc"] == nls.ReturnCode.Success)
    assert_matches_oracle(r512, oracle(po, N, u0, A, B, abstol=1e-8, gmres_orth=po.ORTH_MGS))
    for out in (r512, rmid, rall):
        assert_residuals_consistent(nls, N, out, A, B, 1e-8)


# ----------------------------------------------------------------------------- 4. option sets the kernel implements
TERM = {"safebest": 0, "absnorm": 1, "safe": 2}  # po.TERM_ABS_NORM_SAFE_BEST / TERM_ABS_NORM / TERM_ABS_NORM_SAFE
TERM_CLS = {"safebest": "AbsNormSafeBestTerminationMode", "absnorm": "AbsNormTerminationMode", "safe": "AbsNormSafeTerminationMode"}


@pytest.mark.gpu
@pytest.mark.parametrize("orth", ["mgs", "cgs2"])
@pytest.mark.parametrize("term", ["safebest", "safe", "absnorm"])
def test_orth_and_termination_vs_oracle(nls, ctx, po, orth, term):
    import bench
    N, K = 23, 6
    A, B = bench.ensemble_params(K)
    u0 = start(po, N, K, 0.05)
    tc = getattr(nls, TERM_CLS[term])()
    out = ens_solve(nls, ctx, N, u0, A, B, nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(orth=orth)), abstol=1e-8, termination_condition=tc)
    assert out["launches"] <= 2
    assert_matches_oracle(out, oracle(po, N, u0, A, B, abstol=1e-8, gmres_orth=ORTH[orth], termination=TERM[term]))
    assert_residuals_consistent(nls, N, out, A, B, 1e-8)


@pytest.mark.gpu
def test_eisenstat_walker_forcing_vs_oracle(nls, ctx, po):
    import bench
    N, K = 32, 8
    A, B = bench.ensemble_params(K)
    u0 = start(po, N, K, 0.02)
    alg = nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(orth="mgs"), forcing=nls.EisenstatWalkerForcing2())
    out = ens_solve(nls, ctx, N, u0, A, B, alg, abstol=1e-8)
    ref = oracle(po, N, u0, A, B, abstol=1e-8, gmres_orth=po.ORTH_MGS, forcing=po.FORCING_EW2)
    plain = oracle(po, N, u0, A, B, abstol=1e-8, gmres_orth=po.ORTH_MGS)
    assert not np.array_equal(ref[4], plain[4])      # forcing changes the linear solves
    assert np.all(out["rc"] == nls.ReturnCode.Success)
    assert_matches_oracle(out, ref)
    assert_residuals_consistent(nls, N, out, A, B, 1e-8)


@pytest.mark.gpu
def test_gmres_itmax_inside_the_kernel_vs_oracle(nls, ctx, po):
    """itmax = 40 stops GMRES in most Newton steps (with itmax = 10 the iteration stagnates and runs to maxiters)."""
    import bench
    N, K, itmax = 12, 6, 40
    A, B = bench.ensemble_params(K)
    u0 = start(po, N, K, 0.05)
    out = ens_solve(nls, ctx, N, u0, A, B, nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(orth="cgs2", itmax=itmax)), abstol=1e-9)
    ref = oracle(po, N, u0, A, B, abstol=1e-9, gmres_orth=po.ORTH_CGS2, gmres_itmax=itmax)
    _, _, _, tr = po.OracleProblem.bruss2d(N, A=A[0], B=B[0]).newton(u0[0], po.default_newton_opts(abstol=1e-9, gmres_orth=po.ORTH_CGS2, gmres_itmax=itmax))
    assert sum(t.lin_status == po.LS_MAXITERS for t in tr) >= 2    # GMRES ends on itmax in most Newton steps
    assert np.all(out["rc"] == nls.ReturnCode.Success)
    assert np.all(out["nj"] <= itmax * out["ns"])
    assert np.all(out["nj"] >= itmax * (out["ns"] - 2))
    assert_matches_oracle(out, ref)
    assert_residuals_consistent(nls, N, out, A, B, 1e-9)


@pytest.mark.gpu
def test_explicit_gmres_tolerances_vs_oracle(nls, ctx, po):
    import bench
    N, K = 17, 6
    A, B = bench.ensemble_params(K)
    u0 = start(po, N, K, 0.05)
    out = ens_solve(nls, ctx, N, u0, A, B, nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(orth="mgs", atol=1e-9, rtol=1e-4)), abstol=1e-8)
    ref = oracle(po, N, u0, A, B, abstol=1e-8, gmres_orth=po.ORTH_MGS, gmres_atol=1e-9, gmres_rtol=1e-4)
    inherited = oracle(po, N, u0, A, B, abstol=1e-8, gmres_orth=po.ORTH_MGS)
    assert not np.array_equal(ref[4], inherited[4])
    assert_matches_oracle(out, ref)
    assert_residuals_consistent(nls, N, out, A, B, 1e-8)


@pytest.mark.gpu
def test_wild_starts_best_iterate_rollback(nls, ctx, po):
    """Starts 10^3..10^8 N(0, 1) away from u0, 12 Newton steps: every trajectory ends with MaxIters, and where the last
    iterate is not the best one AbsNormSafeBest returns the best one with its recomputed residual.  The Jacobian there is
    dominated by u^2 ~ 10^16 and nearly singular, so the kernel's iterates and the oracle's part after a few steps: retcodes
    and step counts are compared with the oracle, the iterates with the same kernel in AbsNormSafe mode (which runs the
    same steps and returns the last iterate) and with the extended-precision residual."""
    N, K, maxiters = 8, 48, 12
    rng = np.random.default_rng(7)
    P = po.OracleProblem.bruss2d(N)
    mags = 10.0 ** rng.uniform(3, 8, K)
    u0 = P.u0()[None, :] + mags[:, None] * rng.standard_normal((K, 2 * N * N))
    A, B = np.full(K, 3.4), np.full(K, 1.0)
    opts = dict(abstol=1e-8, gmres_orth=po.ORTH_MGS, maxiters=maxiters)
    rolled = []
    for m in range(K):
        _, _, r, tr = P.newton(u0[m], po.default_newton_opts(**opts))
        if tr[-1].fnorm_inf != r.resid_inf:
            rolled.append(m)
    assert len(rolled) >= 3, rolled
    alg = nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(orth="mgs"))
    best = ens_solve(nls, ctx, N, u0, A, B, alg, abstol=1e-8, maxiters=maxiters)
    last = ens_solve(nls, ctx, N, u0, A, B, alg, abstol=1e-8, maxiters=maxiters, termination_condition=nls.AbsNormSafeTerminationMode())
    ref = oracle(po, N, u0, A, B, **opts)
    for out in (best, last):
        assert np.all(out["rc"] == nls.ReturnCode.MaxIters) and np.array_equal(out["rc"], ref[2]) and np.array_equal(out["ns"], ref[3])
        assert_residuals_consistent(nls, N, out, A, B, 1e-8)
    assert np.array_equal(best["nj"], last["nj"])
    rb = ~np.all(best["u"] == last["u"], axis=1)
    print("rollback in %d of %d trajectories (oracle: %d)" % (rb.sum(), K, len(rolled)))
    assert rb.sum() >= 3
    assert np.all(best["resid"][rb] <= last["resid"][rb])
    assert np.array_equal(best["resid"][~rb], last["resid"][~rb])


@pytest.mark.gpu
def test_near_singular_start(nls, ctx, po):
    """A = -1, u0 = 0: too chaotic to compare iterates; retcodes match the oracle and every reported residual is the
    residual of the returned iterate."""
    N, K = 8, 4
    u0 = np.zeros((K, 2 * N * N))
    A, B = np.full(K, -1.0), 1.0 + 0.01 * np.arange(K)
    out = ens_solve(nls, ctx, N, u0, A, B, nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(orth="mgs")), abstol=1e-8, maxiters=20)
    ref = oracle(po, N, u0, A, B, abstol=1e-8, gmres_orth=po.ORTH_MGS, maxiters=20)
    assert np.array_equal(out["rc"], ref[2]) and np.all(out["rc"] == nls.ReturnCode.MaxIters)
    assert_residuals_consistent(nls, N, out, A, B, 1e-8)


# ----------------------------------------------------------------------------- 5. option sets the kernel does not implement
def _case(N=8, K=2, term=None, orth="mgs", itmax=0, **kw):
    return dict(N=N, K=K, term=term, orth=orth, itmax=itmax, kw=kw)


UNIMPLEMENTED = {
    # loose reltol: these modes stop long before ||f||_inf <= abstol
    "norm": _case(term=("NormTerminationMode", {}), abstol=1e-8, reltol=1e-2),
    "rel": _case(term=("RelTerminationMode", {}), abstol=1e-8, reltol=1e-2),
    "rel_norm": _case(term=("RelNormTerminationMode", {}), abstol=1e-8, reltol=1e-2),
    "rel_norm_safe": _case(term=("RelNormSafeTerminationMode", {}), abstol=1e-8, reltol=1e-2),
    "rel_norm_safe_best": _case(term=("RelNormSafeBestTerminationMode", {}), abstol=1e-8, reltol=1e-2),
    # abstol just under the N = 8 residual floor (1.3e-12 .. 2.3e-12): Abs runs to maxiters, a Safe mode stalls at step 101
    "abs": _case(term=("AbsTerminationMode", {}), abstol=9e-13, maxiters=110),
    # at step 3 ||f||_inf ~ 1.8e-8 <= abstol < ||f||_2 ~ 8e-8
    "l2_abs_norm": _case(term=("AbsNormTerminationMode", {"norm": "l2"}), abstol=3e-8),
    "l2_abs_norm_safe": _case(term=("AbsNormSafeTerminationMode", {"norm": "l2"}), abstol=3e-8),
    "l2_abs_norm_safe_best": _case(term=("AbsNormSafeBestTerminationMode", {"norm": "l2"}), abstol=3e-8),
    # one Arnoldi step per Newton step: steps fall under abstol long before ||f||_inf does (window 5: step ~27, 32: ~54)
    "stall_none": _case(term=("AbsNormSafeTerminationMode", {"max_stalled_steps": None}), itmax=1, abstol=0.02, maxiters=70),
    "stall_5": _case(term=("AbsNormSafeTerminationMode", {"max_stalled_steps": 5}), itmax=1, abstol=0.02, maxiters=70),
    # one classical pass loses orthogonality at N = 32: tens to hundreds more Arnoldi steps than two passes
    "cgs": _case(N=32, orth="cgs", abstol=1e-10),
    "maxtime": _case(abstol=1e-8, maxtime=1e-9),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(UNIMPLEMENTED))
def test_unimplemented_options_match_the_driver(nls, ctx, po, case):
    import bench
    c = UNIMPLEMENTED[case]
    N, K = c["N"], c["K"]
    A, B = bench.ensemble_params(K)
    u0 = start(po, N, K, 0.05)
    kw = dict(c["kw"])
    if c["term"]:
        kw["termination_condition"] = getattr(nls, c["term"][0])(**c["term"][1])
    alg = nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(orth=c["orth"], itmax=c["itmax"]))
    out = ens_solve(nls, ctx, N, u0, A, B, alg, **kw)
    for m in range(K):
        sol = nls.solve(nls.NonlinearProblem(nls.Brusselator2D(N), u0[m].copy(), (A[m], B[m], ALPHA), ctx=ctx), alg, store_trace=False, **kw)
        print("%s m=%d: driver %s nsteps=%d njvp=%d; ensemble %s nsteps=%d njvp=%d" % (
            case, m, nls.ReturnCode.name(sol.retcode), sol.stats.nsteps, sol.stats.njvp, nls.ReturnCode.name(out["rc"][m]), out["ns"][m], out["nj"][m]))
        assert out["rc"][m] == sol.retcode and out["ns"][m] == sol.stats.nsteps and out["nj"][m] == sol.stats.njvp
        assert np.abs(out["u"][m] - sol.u).max() <= RTOL_ROOT * np.abs(sol.u).max()
        assert out["resid"][m] == sol.resid_inf
    assert_residuals_consistent(nls, N, out, A, B, kw["abstol"] if c["term"] is None or "Abs" in c["term"][0] else np.inf)
