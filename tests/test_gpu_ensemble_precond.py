"""Preconditioned ensembles: `EnsembleCache` with `KrylovJL_GMRES(precs = ...)`.

Multigrid on either side is batched: `ens_newton_kernel<ENS_PC_MG_LEFT / RIGHT>` (csrc/ens_batched.cu) runs the V-cycle of
csrc/mg.cu in shared memory inside the one-CTA-per-trajectory kernel.  It is held to

* the single-system preconditioner (`b200_linop_precond`) bit for bit, through `EnsembleCache.precond_apply`, and to the NumPy
  restatement `oracle/mg_numpy.py` to rounding;
* the single-system driver (`nls.solve` of each trajectory alone, same algorithm): retcode and `nsteps` equal, roots to
  RTOL_ROOT, `njvp` to +-1 Arnoldi step per Newton step (the kernel's reductions are ordered differently);
* itself: a second solve, a trajectory alone and a permuted batch give the same bits.

Block-Jacobi, N > 32 and multigrid with an option set the kernel does not cover take the driver trajectory by trajectory and
match it exactly; ILU0 and the AMGs, which need an assembled Jacobian, are refused.  The multigrid hierarchy takes the
problem's A at every setup, so `reinit(cache, u0, p)` with a new A runs exactly what a cache created at that p runs."""
import numpy as np
import pytest

from test_gpu_ensemble import ALPHA, RTOL_ROOT, assert_bit_identical, assert_residuals_consistent, ens_solve, resolve, start

pytestmark = pytest.mark.gpu

SIZES = (3, 9, 12, 16, 27, 31, 32)   # ratio 3 to one cell, 3*3, 2*2*3, 2^4, 3^3, a prime (31 -> 1), the bench size
TERM_CLS = {"absnorm": "AbsNormTerminationMode", "safe": "AbsNormSafeTerminationMode", "safebest": "AbsNormSafeBestTerminationMode"}


def mg_alg(nls, side="right", orth="mgs", ew=False, **gm):
    return nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(orth=orth, precs=nls.Multigrid(side), **gm),
                             forcing=nls.EisenstatWalkerForcing2() if ew else None)


# left preconditioning with the inherited tolerances stops on ||M^-1 f||: tighten GMRES so that the Newton steps still land
OPTIONS = {
    "right": dict(side="right"),
    "left": dict(side="left", atol=1e-13, rtol=1e-9),
    "right_ew": dict(side="right", ew=True),
}


def driver_solve(nls, ctx, N, u0, A, B, alg, **kw):
    K = len(A)
    out = dict(u=np.empty((K, 2 * N * N)), resid=np.empty(K), rc=np.empty(K, np.int32), ns=np.empty(K, np.int32), nj=np.empty(K, np.int32))
    for m in range(K):
        sol = nls.solve(nls.NonlinearProblem(nls.Brusselator2D(N), u0[m].copy(), (A[m], B[m], ALPHA), ctx=ctx), alg, store_trace=False, **kw)
        out["u"][m], out["resid"][m], out["rc"][m], out["ns"][m], out["nj"][m] = sol.u, sol.resid_inf, sol.retcode, sol.stats.nsteps, sol.stats.njvp
    return out


def assert_matches_driver(out, drv):
    assert np.array_equal(out["rc"], drv["rc"]), (out["rc"], drv["rc"])
    assert np.array_equal(out["ns"], drv["ns"]), (out["ns"], drv["ns"])
    scale = np.maximum(np.abs(drv["u"]).max(axis=1), 1e-300)
    err = np.abs(out["u"] - drv["u"]).max(axis=1) / scale
    assert np.all(err <= RTOL_ROOT), err.max()
    assert np.all(np.abs(out["nj"] - drv["nj"]) <= drv["ns"]), (out["nj"], drv["nj"])


def bench_batch(nls, ctx, N, K):
    import bench
    A, B = bench.ensemble_params(K)
    dp = nls._DeviceProblem(ctx, nls.NonlinearProblem(nls.Brusselator2D(N), None, (3.4, 1.0, ALPHA), ctx=ctx))
    return np.tile(dp.u0().to_host(), (K, 1)), A, B


# ----------------------------------------------------------------------------- 1. the V-cycle, bit for bit
@pytest.mark.parametrize("N", SIZES)
@pytest.mark.parametrize("side", ["left", "right"])
def test_vcycle_matches_the_single_system_preconditioner(nls, ctx, po, N, side):
    from oracle import mg_numpy as mgn
    K, n = 4, 2 * N * N
    rng = np.random.default_rng(1000 * N + (side == "left"))
    A = np.array([3.4, 3.55, 3.7, 3.95])
    u = po.OracleProblem.bruss2d(N).u0()[None, :] * (1.0 + 0.05 * rng.standard_normal((K, n)))
    x = rng.standard_normal((K, n))
    cache = nls.EnsembleCache(ctx, N, K, ALPHA, mg_alg(nls, side), abstol=1e-8)
    y = cache.precond_apply(ctx.to_device(u.ravel()), ctx.to_device(A), ctx.to_device(x.ravel())).to_host().reshape(K, n)
    for m in range(K):
        dp = nls._DeviceProblem(ctx, nls.NonlinearProblem(nls.Brusselator2D(N), None, (A[m], 1.0, ALPHA), ctx=ctx))
        du, dx = ctx.to_device(u[m]), ctx.to_device(x[m])
        op = nls.Multigrid(side).linop(dp, du)
        ym = ctx.zeros(n)
        nls.abi.check(ctx.handle, nls.abi.lib().b200_linop_apply(op, dx.ptr, ym.ptr))
        ref = ym.to_host()
        nls.abi.lib().b200_linop_destroy(op)
        assert np.array_equal(y[m], ref), (m, np.abs(y[m] - ref).max())
        mg = mgn.Multigrid(N, 2, u[m], A=A[m], alpha=ALPHA)
        z = mg.vcycle(x[m])
        assert np.abs(y[m] - z).max() <= 1e-11 * np.abs(z).max(), (m, mg.sizes())


def test_precond_apply_refuses_other_ensembles(nls, ctx):
    N, K = 8, 2
    for alg, n in ((nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES()), N), (mg_alg(nls), 33),
                   (nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(precs=nls.BlockJacobi("left"))), N)):
        cache = nls.EnsembleCache(ctx, n, K, ALPHA, alg, abstol=1e-8)
        zz = ctx.zeros(K * 2 * n * n)
        with pytest.raises(nls.abi.B200Error) as e:
            cache.precond_apply(zz, ctx.zeros(K), zz, zz)
        assert e.value.code == nls.abi.ERR_INVALID


# ----------------------------------------------------------------------------- 2. solves against the driver
# Eisenstat-Walker forcing from these starts does not settle at N = 3 and 9: the iterations wander for hundreds of Newton steps
# or run to maxiters, where two solvers that reduce in different orders part ways.  The forcing is held from N = 12 up.
SOLVE_CASES = [(N, option, orth, term) for N in SIZES for option in OPTIONS for orth in ("mgs", "cgs2") for term in TERM_CLS
               if not (option == "right_ew" and N < 12)]


@pytest.mark.parametrize("N,option,orth,term", SOLVE_CASES)
def test_multigrid_batch_matches_the_driver(nls, ctx, po, N, option, orth, term):
    import bench
    K = 8
    A, B = bench.ensemble_params(K)
    u0 = start(po, N, K, 0.02)
    alg = mg_alg(nls, orth=orth, **OPTIONS[option])
    kw = dict(abstol=1e-8, termination_condition=getattr(nls, TERM_CLS[term])())
    out = ens_solve(nls, ctx, N, u0, A, B, alg, **kw)
    assert out["launches"] <= 2                      # one kernel for the whole batch
    assert out["cache"].ctas_per_sm() >= 1
    drv = driver_solve(nls, ctx, N, u0, A, B, alg, **kw)
    print("N=%d %s %s %s: nsteps %s njvp %s (driver %s)" % (N, option, orth, term, out["ns"].tolist(), out["nj"].tolist(), drv["nj"].tolist()))
    assert np.all(out["rc"] == nls.ReturnCode.Success)
    assert_matches_driver(out, drv)
    assert_residuals_consistent(nls, N, out, A, B, 1e-8)


# ----------------------------------------------------------------------------- 3. the work is cut
def test_multigrid_cuts_the_arnoldi_work(nls, ctx):
    N, K = 32, 64
    u0, A, B = bench_batch(nls, ctx, N, K)
    plain = ens_solve(nls, ctx, N, u0, A, B, nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(orth="mgs")), abstol=1e-8)
    mg = ens_solve(nls, ctx, N, u0, A, B, mg_alg(nls), abstol=1e-8)
    print("total njvp: none %d, multigrid right %d; CTAs per SM %d / %d" % (
        plain["nj"].sum(), mg["nj"].sum(), plain["cache"].ctas_per_sm(), mg["cache"].ctas_per_sm()))
    assert np.all(plain["rc"] == nls.ReturnCode.Success) and np.all(mg["rc"] == nls.ReturnCode.Success)
    assert 8 * mg["nj"].sum() <= plain["nj"].sum()
    assert mg["cache"].ctas_per_sm() == plain["cache"].ctas_per_sm() == 2   # the hierarchy fits beside two CTAs per SM
    assert_residuals_consistent(nls, N, mg, A, B, 1e-8)


# ----------------------------------------------------------------------------- 4. routes
ROUTES = {
    "block_jacobi_left": dict(N=8, alg=lambda nls: nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(precs=nls.BlockJacobi("left")))),
    "block_jacobi_right": dict(N=8, alg=lambda nls: nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(precs=nls.BlockJacobi("right")))),
    "multigrid_n33": dict(N=33, alg=lambda nls: mg_alg(nls)),
    "multigrid_rel_norm": dict(N=8, alg=lambda nls: mg_alg(nls, side="left"), term="RelNormTerminationMode", reltol=1e-2),
}


@pytest.mark.parametrize("case", list(ROUTES))
def test_unbatched_preconditioned_sets_match_the_driver(nls, ctx, po, case):
    import bench
    c = ROUTES[case]
    N, K = c["N"], 2
    A, B = bench.ensemble_params(K)
    u0 = start(po, N, K, 0.05)
    kw = dict(abstol=1e-8)
    if "term" in c:
        kw["termination_condition"] = getattr(nls, c["term"])()
        kw["reltol"] = c["reltol"]
    alg = c["alg"](nls)
    out = ens_solve(nls, ctx, N, u0, A, B, alg, **kw)
    assert out["cache"].ctas_per_sm() == 0
    drv = driver_solve(nls, ctx, N, u0, A, B, alg, **kw)
    for m in range(K):
        assert out["rc"][m] == drv["rc"][m] and out["ns"][m] == drv["ns"][m] and out["nj"][m] == drv["nj"][m]
        assert np.abs(out["u"][m] - drv["u"][m]).max() <= RTOL_ROOT * np.abs(drv["u"][m]).max()
        assert out["resid"][m] == drv["resid"][m]
    assert_residuals_consistent(nls, N, out, A, B, 1e-8 if "term" not in c else np.inf)


@pytest.mark.parametrize("precs", ["ILU0", "RugeStubenAMG", "SmoothedAggregationAMG"])
@pytest.mark.parametrize("side", ["left", "right"])
def test_assembled_jacobian_preconditioners_are_refused(nls, ctx, precs, side):
    alg = nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(precs=getattr(nls, precs)(side)))
    with pytest.raises(nls.abi.B200Error) as e:
        nls.EnsembleCache(ctx, 8, 2, ALPHA, alg, abstol=1e-8)
    assert e.value.code == nls.abi.ERR_INVALID


def test_trust_region_is_still_refused(nls, ctx):
    alg = nls.TrustRegion(linsolve=nls.KrylovJL_GMRES(precs=nls.Multigrid("right")))
    with pytest.raises(nls.abi.B200Error) as e:
        nls.EnsembleCache(ctx, 8, 2, ALPHA, alg, abstol=1e-8)
    assert e.value.code == nls.abi.ERR_INVALID


# ----------------------------------------------------------------------------- 5. deferral
@pytest.mark.parametrize("side", ["left", "right"])
def test_deferred_trajectories_match_the_driver_exactly(nls, ctx, po, monkeypatch, side):
    """A 4-column basis slab is below what multigrid GMRES needs (about 10 Arnoldi steps): the trajectories that outgrow it are
    redone by the general driver and carry its bits; the others carry the bits of the full-slab batch."""
    import bench
    N, K = 16, 8
    A, B = bench.ensemble_params(K)
    u0 = start(po, N, K, 0.1)
    alg = mg_alg(nls, **OPTIONS[side])
    full = ens_solve(nls, ctx, N, u0, A, B, alg, abstol=1e-8)
    drv = driver_solve(nls, ctx, N, u0, A, B, alg, abstol=1e-8)
    monkeypatch.setenv("B200_ENS_BASIS_COLUMNS", "4")
    capped = ens_solve(nls, ctx, N, u0, A, B, alg, abstol=1e-8)
    monkeypatch.delenv("B200_ENS_BASIS_COLUMNS")

    def same(a, b, m):
        return all(np.array_equal(a[k][m], b[k][m]) for k in ("u", "resid", "rc", "ns", "nj"))

    as_full = np.array([same(capped, full, m) for m in range(K)])
    as_drv = np.array([same(capped, drv, m) for m in range(K)])
    print("%s: %d of %d trajectories deferred" % (side, int((as_drv & ~as_full).sum()), K))
    assert np.all(as_full | as_drv), (as_full, as_drv)
    assert np.any(as_drv & ~as_full)
    assert_matches_driver(full, drv)
    assert_residuals_consistent(nls, N, capped, A, B, 1e-8)


# ----------------------------------------------------------------------------- 6. determinism
@pytest.mark.parametrize("option", list(OPTIONS))
def test_multigrid_batch_is_deterministic(nls, ctx, option):
    N, K = 32, 96
    u0, A, B = bench_batch(nls, ctx, N, K)
    alg = mg_alg(nls, **OPTIONS[option])
    out = ens_solve(nls, ctx, N, u0, A, B, alg, abstol=1e-8)
    assert np.all(out["rc"] == nls.ReturnCode.Success)
    assert_bit_identical(out, resolve(nls, ctx, out))
    for m in (0, 37, K - 1):
        alone = ens_solve(nls, ctx, N, u0[m:m + 1], A[m:m + 1], B[m:m + 1], alg, abstol=1e-8)
        assert_bit_identical(out, alone, slice(m, m + 1))
    perm = np.random.default_rng(K).permutation(K)
    permuted = ens_solve(nls, ctx, N, u0[perm], A[perm], B[perm], alg, abstol=1e-8)
    assert_bit_identical(out, permuted, perm)


# ----------------------------------------------------------------------------- 7. the hierarchy follows the problem's A
@pytest.mark.parametrize("dim,N", [(2, 16), (3, 8)])
@pytest.mark.parametrize("side", ["left", "right"])
def test_reinit_with_new_parameters_rebuilds_the_hierarchy(nls, ctx, dim, N, side):
    f = nls.Brusselator2D(N) if dim == 2 else nls.Brusselator3D(N)
    u0 = nls._DeviceProblem(ctx, nls.NonlinearProblem(f, None, (3.4, 1.0, ALPHA), ctx=ctx)).u0().to_host()
    alg = mg_alg(nls, side, atol=1e-13, rtol=1e-9) if side == "left" else mg_alg(nls, side)
    old = nls.init(nls.NonlinearProblem(f, u0.copy(), (3.4, 1.0, ALPHA), ctx=ctx), alg, abstol=1e-8)
    old.solve()
    old.reinit(u0.copy(), p=(3.7, 1.02, ALPHA))
    a = old.solve()
    b = nls.init(nls.NonlinearProblem(f, u0.copy(), (3.7, 1.02, ALPHA), ctx=ctx), alg, abstol=1e-8).solve()
    assert b.retcode == nls.ReturnCode.Success
    assert vars(a.stats) == vars(b.stats)
    assert [t.lin_iters for t in a.trace] == [t.lin_iters for t in b.trace]
    assert [t.fnorm_inf for t in a.trace] == [t.fnorm_inf for t in b.trace]
    assert a.resid_inf == b.resid_inf
    assert np.array_equal(np.asarray(a.u), np.asarray(b.u))
