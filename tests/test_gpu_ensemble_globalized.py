"""Globalised ensembles: `TrustRegion(linsolve = KrylovJL_GMRES())` (Dogleg, six radius schemes) and
`NewtonRaphson(linsolve = KrylovJL_GMRES(), linesearch = BackTracking())` batched inside the one-CTA-per-trajectory kernel
(`ens_newton_kernel<ENS_PC_NONE, ENS_GL_TRUST_REGION / ENS_GL_LINESEARCH>`, csrc/ens_batched.cu).

References:

* the per-trajectory C oracle (`po.ensemble_solve`, `OracleProblem.newton`), which restates newton.cu's dogleg, trust-region
  step and BackTracking: retcode and `nsteps` equal, roots to RTOL_ROOT, `njvp` to +-2 Arnoldi steps per Newton step;
* the single-system CUDA driver (`nls.solve` of one trajectory) for the option sets the kernel does not cover (Bastin, the L2
  termination norm, N > 32) and for deferred trajectories, which `b200_ens_solve` routes to it: equal bit for bit;
* the kernel itself: a second solve, a trajectory alone and a permuted batch give the same bits.

The far start is 30 u0 at N = 12: from there the trust region rejects steps and cuts them at the radius, and BackTracking
shortens steps (one trajectory of the batch ends Stalled).  The oracle-only tests at the top check that on the CPU.  Every
row-walk geometry up to N = 32 is compared with the oracle from a start near u0.  From 10 u0 + 0.1 at N = 32 GMRES needs
500-600 Arnoldi steps per Newton step, past the default 512-column slab, and the oracle about a minute per trajectory; that
start is left to tools/ens_globalized_bench.py."""
import numpy as np
import pytest

from test_gpu_ensemble import (ALPHA, GEOMETRY_N, ORTH, RTOL_ROOT, TERM, TERM_CLS, assert_bit_identical, assert_matches_oracle,
                               assert_residuals_consistent, ens_solve, oracle, resolve, start)
from test_gpu_ensemble_precond import assert_matches_driver, driver_solve

SCHEMES = ("Simple", "NLsolve", "NocedalWright", "Hei", "Yuan", "Fan")   # the schemes the C oracle restates
TR_CODE = {"Simple": 0, "NLsolve": 1, "NocedalWright": 2, "Hei": 3, "Yuan": 4, "Fan": 5, "Bastin": 6}  # abi.TR_* / po.TR_*
GLOB_TR, GLOB_LS = 1, 2   # po.GLOB_TRUST_REGION / GLOB_LINESEARCH


def far_start(po, N, K, scale=30.0):
    return np.tile(scale * po.OracleProblem.bruss2d(N).u0(), (K, 1))


# BackTracking from 30 u0 shortens steps to alpha ~ 1e-25 and its path is chaotic: the oracle's own MGS and CGS2 runs take
# 30 / 36 / 55 / 32 and 30 / 30 / 200 / 40 Newton steps, so reduction order alone changes them.  From 8 u0 it still takes
# alpha < 1 (down to 0.05) and both orthogonalisations give the same steps: the parity tests start there.
LS_SCALE = 8.0


def tr_alg(nls, scheme="Simple", orth="mgs", ew=False, itmax=0, **tr):
    alg = nls.TrustRegion(linsolve=nls.KrylovJL_GMRES(orth=orth, itmax=itmax), radius_update_scheme=getattr(nls.RadiusUpdateSchemes, scheme), **tr)
    if ew:
        alg.forcing = nls.EisenstatWalkerForcing2()
    return alg


def ls_alg(nls, orth="mgs", **bt):
    return nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(orth=orth), linesearch=nls.BackTracking(**bt))


def tr_opts(scheme="Simple", **kw):
    return dict(globalization=GLOB_TR, tr_scheme=TR_CODE[scheme], **kw)


def ls_opts(**kw):
    return dict(globalization=GLOB_LS, **kw)


def traces(po, N, u0, A, B, **opts):
    out = []
    for m in range(len(A)):
        _, _, r, tr = po.OracleProblem.bruss2d(N, A=A[m], B=B[m]).newton(u0[m], po.default_newton_opts(**opts))
        out.append((r, tr))
    return out


# ----------------------------------------------------------------------------- the inputs exercise what they claim (no GPU)
def test_oracle_far_start_exercises_every_dogleg_outcome(po):
    """30 u0 at N = 12: the trust region rejects steps, takes Newton steps strictly inside the radius, and takes steps that end
    on it (the Cauchy direction cut at the radius, or the dogleg)."""
    import bench
    N, K = 12, 2
    A, B = bench.ensemble_params(K)
    u0 = far_start(po, N, K)
    rejected = inside = on_radius = 0
    for scheme in SCHEMES:
        for r, tr in traces(po, N, u0, A, B, abstol=1e-8, gmres_orth=po.ORTH_CGS2, maxiters=200, **tr_opts(scheme)):
            assert r.retcode == po.RC_SUCCESS, (scheme, r.retcode)
            for prev, t in zip(tr, tr[1:]):   # the radius a step was taken with is the one the previous step left
                if not t.accepted:
                    rejected += 1
                elif t.step_norm2 < prev.trust_radius * (1 - 1e-6):
                    inside += 1
                elif abs(t.step_norm2 - prev.trust_radius) <= 1e-6 * prev.trust_radius:
                    on_radius += 1
    print("rejected %d, inside the radius %d, on the radius %d" % (rejected, inside, on_radius))
    assert rejected > 0 and inside > 0 and on_radius > 0


def test_oracle_far_start_backtracks(po):
    """30 u0 at N = 12: BackTracking takes alpha < 1 on some step, and one trajectory of the batch ends Stalled."""
    import bench
    N, K = 12, 4
    A, B = bench.ensemble_params(K)
    res = traces(po, N, far_start(po, N, K), A, B, abstol=1e-8, gmres_orth=po.ORTH_CGS2, maxiters=200, **ls_opts())
    alphas = [t.trust_radius for _, tr in res for t in tr]   # the trace's trust_radius slot holds alpha for a line search
    rcs = [r.retcode for r, _ in res]
    print("alpha range %.3g .. %.3g; retcodes %s" % (min(alphas), max(alphas), rcs))
    assert min(alphas) < 1.0
    assert po.RC_SUCCESS in rcs and po.RC_STALLED in rcs


# ----------------------------------------------------------------------------- 1. parity with the oracle
# every scheme with MGS / SafeBest, CGS2 / AbsNorm and MGS / Safe from the far start at N = 12
MODES = (("mgs", "safebest"), ("cgs2", "absnorm"), ("mgs", "safe"))
TR_CASES = [(12, s, o, t) for s in SCHEMES for o, t in MODES]


@pytest.mark.gpu
@pytest.mark.parametrize("N,scheme,orth,term", TR_CASES)
def test_trust_region_vs_oracle(nls, ctx, po, N, scheme, orth, term):
    import bench
    K = 4
    A, B = bench.ensemble_params(K)
    u0 = far_start(po, N, K)
    kw = dict(abstol=1e-8, maxiters=200, termination_condition=getattr(nls, TERM_CLS[term])())
    out = ens_solve(nls, ctx, N, u0, A, B, tr_alg(nls, scheme, orth), **kw)
    assert out["launches"] <= 2                      # one kernel for the whole batch
    ref = oracle(po, N, u0, A, B, abstol=1e-8, maxiters=200, gmres_orth=ORTH[orth], termination=TERM[term], **tr_opts(scheme))
    print("N=%d %s %s %s: rc %s nsteps %s njvp %s (oracle %s)" % (N, scheme, orth, term, out["rc"].tolist(), out["ns"].tolist(), out["nj"].tolist(), ref[4].tolist()))
    assert_matches_oracle(out, ref)
    assert_residuals_consistent(nls, N, out, A, B, 1e-8)


LS_CASES = [(12, o, t) for o, t in MODES]


@pytest.mark.gpu
@pytest.mark.parametrize("N,orth,term", LS_CASES)
def test_backtracking_vs_oracle(nls, ctx, po, N, orth, term):
    import bench
    K = 4
    A, B = bench.ensemble_params(K)
    u0 = far_start(po, N, K, LS_SCALE)
    r, tr = traces(po, N, u0[:1], A[:1], B[:1], abstol=1e-8, gmres_orth=ORTH[orth], **ls_opts())[0]
    assert min(t.trust_radius for t in tr) < 1.0     # the line search shortens a step
    kw = dict(abstol=1e-8, maxiters=200, termination_condition=getattr(nls, TERM_CLS[term])())
    out = ens_solve(nls, ctx, N, u0, A, B, ls_alg(nls, orth), **kw)
    assert out["launches"] <= 2
    ref = oracle(po, N, u0, A, B, abstol=1e-8, maxiters=200, gmres_orth=ORTH[orth], termination=TERM[term], **ls_opts())
    print("N=%d %s %s: rc %s nsteps %s (oracle rc %s nsteps %s)" % (N, orth, term, out["rc"].tolist(), out["ns"].tolist(), ref[2].tolist(), ref[3].tolist()))
    assert_matches_oracle(out, ref)
    assert_residuals_consistent(nls, N, out, A, B, 1e-8)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [N for N in GEOMETRY_N if N <= 32])
@pytest.mark.parametrize("kind", ["trust_region", "backtracking"])
def test_geometry_vs_oracle(nls, ctx, po, N, kind):
    import bench
    K = 2
    A, B = bench.ensemble_params(K)
    u0 = start(po, N, K, 0.03)
    alg, opts = (tr_alg(nls), tr_opts()) if kind == "trust_region" else (ls_alg(nls), ls_opts())
    out = ens_solve(nls, ctx, N, u0, A, B, alg, abstol=1e-8)
    assert out["launches"] <= 2
    assert np.all(out["rc"] == nls.ReturnCode.Success)
    assert_matches_oracle(out, oracle(po, N, u0, A, B, abstol=1e-8, gmres_orth=po.ORTH_MGS, **opts))
    assert_residuals_consistent(nls, N, out, A, B, 1e-8)


@pytest.mark.gpu
def test_trust_region_with_one_arnoldi_step_per_newton_step(nls, ctx, po):
    """itmax = 1: the basis slab has two columns, which the dogleg's scratch vectors reuse."""
    import bench
    N, K = 8, 4
    A, B = bench.ensemble_params(K)
    u0 = start(po, N, K, 0.05)
    out = ens_solve(nls, ctx, N, u0, A, B, tr_alg(nls, itmax=1), abstol=1e-8, maxiters=60)
    assert out["launches"] <= 2
    ref = oracle(po, N, u0, A, B, abstol=1e-8, maxiters=60, gmres_orth=po.ORTH_MGS, gmres_itmax=1, **tr_opts())
    assert np.array_equal(out["rc"], ref[2]) and np.array_equal(out["ns"], ref[3])
    assert np.all(out["nj"] == out["ns"])
    assert_residuals_consistent(nls, N, out, A, B, 1e-8 if np.all(out["rc"] == nls.ReturnCode.Success) else np.inf)


# ----------------------------------------------------------------------------- 2. Eisenstat-Walker forcing
@pytest.mark.gpu
def test_eisenstat_walker_forcing_with_trust_region(nls, ctx, po):
    """A rejected step keeps fu, so eta follows rnorm_prev <- rnorm on it: the kernel re-runs GMRES with that eta.  From 2 u0
    (two rejected steps per trajectory; from 30 u0 the forced path is as chaotic as BackTracking's)."""
    import bench
    N, K = 12, 4
    A, B = bench.ensemble_params(K)
    u0 = far_start(po, N, K, 2.0)
    out = ens_solve(nls, ctx, N, u0, A, B, tr_alg(nls, ew=True), abstol=1e-8, maxiters=200)
    ref = oracle(po, N, u0, A, B, abstol=1e-8, maxiters=200, gmres_orth=po.ORTH_MGS, forcing=po.FORCING_EW2, **tr_opts())
    plain = oracle(po, N, u0, A, B, abstol=1e-8, maxiters=200, gmres_orth=po.ORTH_MGS, **tr_opts())
    assert not np.array_equal(ref[4], plain[4])      # forcing changes the linear solves
    r, tr = traces(po, N, u0[:1], A[:1], B[:1], abstol=1e-8, maxiters=200, gmres_orth=po.ORTH_MGS, forcing=po.FORCING_EW2, **tr_opts())[0]
    assert any(not t.accepted for t in tr)           # with rejected steps
    assert_matches_oracle(out, ref)
    assert_residuals_consistent(nls, N, out, A, B, 1e-8)


# ----------------------------------------------------------------------------- 3. failure retcodes in mixed batches
def mixed_start(po, N, K, scale=30.0):
    """Even trajectories from the reference u0 (a few full Newton steps), odd ones from scale u0."""
    u0 = np.tile(po.OracleProblem.bruss2d(N).u0(), (K, 1))
    u0[1::2] = far_start(po, N, K, scale)[1::2]
    return u0


FAILURES = {
    "shrink_threshold": dict(alg=lambda nls: tr_alg(nls, max_shrink_times=2), opts=tr_opts(max_shrink_times=2), kw={}, rc="ShrinkThresholdExceeded"),
    "linesearch_failed": dict(alg=lambda nls: ls_alg(nls, maxiters=1), opts=ls_opts(ls_maxiters=1), kw={}, rc="InternalLineSearchFailed"),
    "maxiters_tr": dict(alg=lambda nls: tr_alg(nls), opts=tr_opts(), kw=dict(maxiters=10), rc="MaxIters"),
    "maxiters_ls": dict(alg=lambda nls: ls_alg(nls), opts=ls_opts(), kw=dict(maxiters=5), rc="MaxIters", scale=LS_SCALE),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(FAILURES))
def test_failure_retcodes_in_mixed_batches(nls, ctx, po, case):
    import bench
    c = FAILURES[case]
    N, K = 12, 6
    A, B = bench.ensemble_params(K)
    u0 = mixed_start(po, N, K, c.get("scale", 30.0))
    kw = dict(abstol=1e-8, **c["kw"])
    out = ens_solve(nls, ctx, N, u0, A, B, c["alg"](nls), **kw)
    ref = oracle(po, N, u0, A, B, gmres_orth=po.ORTH_MGS, **kw, **c["opts"])
    print("%s: rc %s (oracle %s) nsteps %s (oracle %s)" % (case, out["rc"].tolist(), ref[2].tolist(), out["ns"].tolist(), ref[3].tolist()))
    fail = getattr(nls.ReturnCode, c["rc"])
    assert np.any(ref[2] == fail) and np.any(ref[2] == nls.ReturnCode.Success)   # a mixed batch
    assert out["launches"] <= 2
    assert_matches_oracle(out, ref)
    assert_residuals_consistent(nls, N, out, A, B, np.inf)


# ----------------------------------------------------------------------------- 4. determinism
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["trust_region", "backtracking"])
def test_globalized_batch_is_deterministic(nls, ctx, po, kind):
    """The far start at N = 12 (rejected, cut and backtracked steps; GMRES never outgrows the slab there)."""
    import bench
    N, K = 12, 96
    A, B = bench.ensemble_params(K)
    u0 = far_start(po, N, K)
    alg = tr_alg(nls) if kind == "trust_region" else ls_alg(nls)
    out = ens_solve(nls, ctx, N, u0, A, B, alg, abstol=1e-8, maxiters=200)
    assert out["launches"] <= 2
    assert np.any(out["rc"] == nls.ReturnCode.Success)
    assert_residuals_consistent(nls, N, out, A, B, 1e-8)
    assert_bit_identical(out, resolve(nls, ctx, out))
    for m in (0, 37, K - 1):
        alone = ens_solve(nls, ctx, N, u0[m:m + 1], A[m:m + 1], B[m:m + 1], alg, abstol=1e-8, maxiters=200)
        assert_bit_identical(out, alone, slice(m, m + 1))
    perm = np.random.default_rng(K).permutation(K)
    permuted = ens_solve(nls, ctx, N, u0[perm], A[perm], B[perm], alg, abstol=1e-8, maxiters=200)
    assert_bit_identical(out, permuted, perm)


# ----------------------------------------------------------------------------- 5. occupancy
@pytest.mark.gpu
def test_globalized_kernels_keep_two_ctas_per_sm(nls, ctx):
    N, K = 32, 4
    for alg in (nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(orth="mgs")), tr_alg(nls), tr_alg(nls, "Yuan"), ls_alg(nls)):
        assert nls.EnsembleCache(ctx, N, K, ALPHA, alg, abstol=1e-8).ctas_per_sm() == 2


# ----------------------------------------------------------------------------- 6. deferral
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["trust_region", "backtracking"])
def test_deferred_globalized_trajectories_match_the_driver_exactly(nls, ctx, po, monkeypatch, kind):
    """A 2-column basis slab is far below what unpreconditioned GMRES needs: every trajectory is redone by the general driver
    and carries its bits."""
    import bench
    N, K = 16, 4
    A, B = bench.ensemble_params(K)
    u0 = start(po, N, K, 0.1)
    alg = tr_alg(nls) if kind == "trust_region" else ls_alg(nls)
    drv = driver_solve(nls, ctx, N, u0, A, B, alg, abstol=1e-8)
    monkeypatch.setenv("B200_ENS_BASIS_COLUMNS", "2")
    capped = ens_solve(nls, ctx, N, u0, A, B, alg, abstol=1e-8)
    monkeypatch.delenv("B200_ENS_BASIS_COLUMNS")
    for key in ("u", "resid", "rc", "ns", "nj"):
        assert np.array_equal(capped[key], drv[key]), key
    full = ens_solve(nls, ctx, N, u0, A, B, alg, abstol=1e-8)
    assert_matches_driver(full, drv)
    assert_residuals_consistent(nls, N, capped, A, B, 1e-8)


# ----------------------------------------------------------------------------- 7. routes to the driver
ROUTES = {
    "bastin": dict(N=8, alg=lambda nls: tr_alg(nls, "Bastin")),
    "tr_l2_norm": dict(N=8, alg=lambda nls: tr_alg(nls), term=("AbsNormSafeBestTerminationMode", {"norm": "l2"}), abstol=3e-8),
    "ls_l2_norm": dict(N=8, alg=lambda nls: ls_alg(nls), term=("AbsNormSafeBestTerminationMode", {"norm": "l2"}), abstol=3e-8),
    "tr_n33": dict(N=33, alg=lambda nls: tr_alg(nls)),
    "ls_n33": dict(N=33, alg=lambda nls: ls_alg(nls)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(ROUTES))
def test_unbatched_globalized_sets_match_the_driver(nls, ctx, po, case):
    import bench
    c = ROUTES[case]
    N, K = c["N"], 2
    A, B = bench.ensemble_params(K)
    u0 = start(po, N, K, 0.05)
    kw = dict(abstol=c.get("abstol", 1e-8))
    if "term" in c:
        kw["termination_condition"] = getattr(nls, c["term"][0])(**c["term"][1])
    alg = c["alg"](nls)
    out = ens_solve(nls, ctx, N, u0, A, B, alg, **kw)
    assert out["cache"].ctas_per_sm() == 0
    drv = driver_solve(nls, ctx, N, u0, A, B, alg, **kw)
    for m in range(K):
        assert out["rc"][m] == drv["rc"][m] and out["ns"][m] == drv["ns"][m] and out["nj"][m] == drv["nj"][m]
        assert np.abs(out["u"][m] - drv["u"][m]).max() <= RTOL_ROOT * np.abs(drv["u"][m]).max()
        assert out["resid"][m] == drv["resid"][m]


# ----------------------------------------------------------------------------- 8. refusals
REFUSED = {
    "tr_block_jacobi_left": lambda nls: nls.TrustRegion(linsolve=nls.KrylovJL_GMRES(precs=nls.BlockJacobi("left"))),
    "tr_block_jacobi_right": lambda nls: nls.TrustRegion(linsolve=nls.KrylovJL_GMRES(precs=nls.BlockJacobi("right"))),
    "ls_multigrid_left": lambda nls: nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(precs=nls.Multigrid("left")), linesearch=nls.BackTracking()),
    "ls_multigrid_right": lambda nls: nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(precs=nls.Multigrid("right")), linesearch=nls.BackTracking()),
    "pseudo_transient": lambda nls: nls.PseudoTransient(linsolve=nls.KrylovJL_GMRES()),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(REFUSED))
def test_refused_ensembles(nls, ctx, case):
    with pytest.raises(nls.abi.B200Error) as e:
        nls.EnsembleCache(ctx, 8, 2, ALPHA, REFUSED[case](nls), abstol=1e-8)
    assert e.value.code == nls.abi.ERR_INVALID


# ----------------------------------------------------------------------------- 9. end to end
@pytest.mark.gpu
def test_solve_ensemble_problem_with_trust_region(nls, ctx, po):
    import bench
    N, K = 12, 4
    A, B = bench.ensemble_params(K)
    u0 = far_start(po, N, K)
    prob = nls.NonlinearProblem(nls.Brusselator2D(N), u0[0].copy(), (A[0], B[0], ALPHA), ctx=ctx)
    pf = lambda pr, i, rep: nls.remake(pr, p=(A[i - 1], B[i - 1], ALPHA))  # noqa: E731
    es = nls.solve(nls.EnsembleProblem(prob, prob_func=pf), nls.TrustRegion(linsolve=nls.KrylovJL_GMRES()), nls.EnsembleB200(),
                   trajectories=K, abstol=1e-8)
    uo, _, rco, nso, _, _ = oracle(po, N, u0, A, B, abstol=1e-8, gmres_orth=po.ORTH_CGS2, **tr_opts())
    assert np.array_equal(es.retcodes, rco) and np.array_equal(es.nsteps, nso)
    assert np.all(es.retcodes == nls.ReturnCode.Success)
    assert np.abs(es.u - uo).max() <= RTOL_ROOT * np.abs(uo).max()
