"""GPU parity tests (run with `-m gpu` on an H100): every kernel family through the C ABI against the CPU oracle
on the same seeded inputs, plus the committed golden fixtures.  Tolerances are stated per test; integer / index work is
bit-exact.  Floating point: the reference arithmetic is Float64 throughout; differences come only from FMA contraction
and reduction order, so 1e-12 relative (scaled by the vector's max) is the bar for single kernels, 1e-6 relative on
roots (BASELINE.json north_star: "residual match to the CPU reference within rtol=1e-6")."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

RTOL_KERNEL = 1e-12
RTOL_ROOT = 1e-6


def close(a, b, rtol=RTOL_KERNEL):
    a, b = np.asarray(a), np.asarray(b)
    scale = max(np.abs(b).max(), 1e-300)
    return np.abs(a - b).max() <= rtol * scale


def make(nls, ctx, po, kind, N=None, n=None, p=None):
    """(device problem wrapper, oracle problem, NonlinearProblem) for one of the built-in problems."""
    if kind == "bruss2d":
        f, P, pp = nls.Brusselator2D(N), po.OracleProblem.bruss2d(N), (3.4, 1.0, 10.0)
    elif kind == "bruss3d":
        f, P, pp = nls.Brusselator3D(N), po.OracleProblem.bruss3d(N), (3.4, 1.0, 10.0)
    elif kind == "quadratic":
        f, P, pp = nls.QuadraticFunction(n), po.OracleProblem.quadratic(n, 2.0), 2.0
    else:
        f, P, pp = nls.TridiagQuadFunction(len(p)), po.OracleProblem.tridiag_quad(p), p
    prob = nls.NonlinearProblem(f, None, pp, ctx=ctx)
    return nls._DeviceProblem(ctx, prob), P, prob


# ----------------------------------------------------------------------------- vector ops (b5 surface)
def test_vector_ops(nls, ctx):
    rng = np.random.default_rng(0)
    for n in (1, 7, 1000, 123457):
        x, y = rng.standard_normal(n), rng.standard_normal(n)
        dx, dy = ctx.to_device(x), ctx.to_device(y)
        assert abs(dx.dot(dy) - x @ y) <= 1e-12 * (np.abs(x) @ np.abs(y))
        assert abs(dx.norm(2) - np.linalg.norm(x)) <= 1e-13 * np.linalg.norm(x)
        assert dx.norm(np.inf) == np.abs(x).max()
        z = dy.copy().axpy(0.5, dx)
        assert np.allclose(z.to_host(), y + 0.5 * x, rtol=1e-15, atol=1e-15)
        assert np.array_equal(dx.copy().scal(-1.0).to_host(), -x)
        out = C.c_double()
        nls.abi.check(ctx.handle, nls.abi.lib().b200_diffnrm2(ctx.handle, n, dx.ptr, dy.ptr, C.byref(out)))
        assert abs(out.value - np.linalg.norm(x - y)) <= 1e-13 * np.linalg.norm(x - y) + 1e-300
        mn, mx = C.c_double(), C.c_double()
        nls.abi.check(ctx.handle, nls.abi.lib().b200_extrema(ctx.handle, n, dx.ptr, C.byref(mn), C.byref(mx)))
        assert (mn.value, mx.value) == (x.min(), x.max())
        eq = C.c_int32()
        dx2 = dx.copy()  # held in a name: a temporary would be freed before the call reads it
        nls.abi.check(ctx.handle, nls.abi.lib().b200_equal(ctx.handle, n, dx.ptr, dx2.ptr, C.byref(eq)))
        assert eq.value == 1
    xn = np.array([1.0, np.nan, 3.0])
    assert not np.isfinite(ctx.to_device(xn).norm(np.inf))  # non-finite propagates (termination_conditions.jl:256)


# ----------------------------------------------------------------------------- residual / JVP / VJP (a1, a2)
@pytest.mark.parametrize("kind,N", [("bruss2d", 8), ("bruss2d", 32), ("bruss2d", 33), ("bruss3d", 6), ("bruss3d", 16), ("bruss3d", 19),
                                     ("bruss3d", 24), ("bruss3d", 26), ("bruss3d", 50)])  # N >= 24, even: the halo-tile kernels (26: ragged last chunk)
def test_residual_jvp_vjp(nls, ctx, po, kind, N):
    dp, P, _ = make(nls, ctx, po, kind, N=N)
    rng = np.random.default_rng(N)
    u = P.u0(1) + 0.1 * rng.standard_normal(P.n)
    v = rng.standard_normal(P.n)
    du, dv = ctx.to_device(u), ctx.to_device(v)
    assert close(dp.u0(1).to_host(), P.u0(1), 1e-14)
    assert close(dp.residual(du).to_host(), P.residual(u))
    assert close(dp.jvp(du, dv).to_host(), P.jvp(u, v))
    assert close(dp.vjp(du, dv).to_host(), P.vjp(u, v))
    f, Jv = dp.residual_jvp(du, dv)
    assert close(f.to_host(), P.residual(u)) and close(Jv.to_host(), P.jvp(u, v))
    # fused finite-difference JVP: same step as the oracle's FiniteDiff restatement -> tight; and close to the exact tangent
    fd = dp.jvp(du, dv, fd=True).to_host()
    assert close(fd, P.jvp_fd(u, v), 1e-6)
    assert close(fd, P.jvp(u, v), 1e-4)


def test_residual_golden(nls, ctx, po, golden):
    for N in (8, 32):
        dp, P, _ = make(nls, ctx, po, "bruss2d", N=N)
        u0 = ctx.to_device(golden["u0_%d" % N])
        assert close(dp.residual(u0).to_host(), golden["f0_%d" % N])
        assert close(dp.jvp(u0, ctx.to_device(golden["v_%d" % N])).to_host(), golden["Jv_%d" % N])
        assert close(dp.vjp(u0, ctx.to_device(golden["v_%d" % N])).to_host(), golden["JTv_%d" % N])


def test_small_problems(nls, ctx, po, golden):
    rng = np.random.default_rng(5)
    dp, P, _ = make(nls, ctx, po, "quadratic", n=1000)
    u, v = rng.standard_normal(1000), rng.standard_normal(1000)
    assert close(dp.residual(ctx.to_device(u)).to_host(), P.residual(u))
    assert close(dp.jvp(ctx.to_device(u), ctx.to_device(v)).to_host(), P.jvp(u, v))
    p = golden["tridiag_p"]
    dp, P, _ = make(nls, ctx, po, "tridiag", p=p)
    u, v = rng.standard_normal(100), rng.standard_normal(100)
    assert close(dp.residual(ctx.to_device(u)).to_host(), P.residual(u))
    assert close(dp.jvp(ctx.to_device(u), ctx.to_device(v)).to_host(), P.jvp(u, v))
    assert close(dp.vjp(ctx.to_device(u), ctx.to_device(v)).to_host(), P.vjp(u, v))


def test_3d_slices_equal_2d(nls, ctx, po):
    # SURVEY.md §A.2: z-independent data -> each k-slice of the 3D result equals the 2D result bit for bit
    N = 20
    d2, P2, _ = make(nls, ctx, po, "bruss2d", N=N)
    d3, P3, _ = make(nls, ctx, po, "bruss3d", N=N)
    rng = np.random.default_rng(2)
    v2 = rng.standard_normal(P2.n)
    v3 = np.concatenate([np.tile(v2[:N * N], N), np.tile(v2[N * N:], N)])
    f2 = d2.residual(d2.u0()).to_host()
    f3 = d3.residual(d3.u0(0)).to_host()
    J2 = d2.jvp(d2.u0(), ctx.to_device(v2)).to_host()
    J3 = d3.jvp(d3.u0(0), ctx.to_device(v3)).to_host()
    for k in (0, 1, N // 2, N - 1):
        for s in range(2):
            sl3 = slice(s * N ** 3 + k * N * N, s * N ** 3 + (k + 1) * N * N)
            sl2 = slice(s * N * N, (s + 1) * N * N)
            assert np.array_equal(f3[sl3], f2[sl2])
            assert np.array_equal(J3[sl3], J2[sl2])


# ----------------------------------------------------------------------------- GMRES (a3)
@pytest.mark.parametrize("orth", ["mgs", "cgs", "cgs2"])
def test_gmres_vs_oracle(nls, ctx, po, orth):
    N = 12
    dp, P, _ = make(nls, ctx, po, "bruss2d", N=N)
    u = P.u0()
    b = P.residual(u)
    code = {"mgs": po.ORTH_MGS, "cgs": po.ORTH_CGS, "cgs2": po.ORTH_CGS2}[orth]
    xo, so, ho = po.gmres(b, prob=P, u=u, opts=po.default_gmres_opts(atol=1e-10, rtol=1e-10, orth=code), want_hessenberg=200000)
    gm = nls.GmresSolver(ctx, P.n, nls.KrylovJL_GMRES(orth=orth, check_every=5), atol=1e-10, rtol=1e-10, keep_hessenberg=200000)
    J = nls.JacobianOperator(dp, ctx.to_device(u))
    x, st = gm.solve(J, ctx.to_device(b))
    assert st.status == nls.abi.LS_SOLVED == so.status
    assert abs(st.iters - so.iters) <= 1  # reduction order may move the stopping test by one step at the margin
    assert abs(st.rnorm0 - so.rnorm0) <= 1e-12 * so.rnorm0
    assert close(x.to_host(), xo, 1e-7)
    # EVERY Hessenberg column both runs produced, column by column (k + 1 entries each, relative to the column's largest
    # entry): the first 40 to 1e-8, all but the last six to 1e-6.  The last columns of a solve driven to rtol 1e-10 are built
    # from vectors whose norm before normalisation is ~1e-7 of the operator's scale — rounding differences between two
    # reduction orders are amplified by that factor there (measured: 1e-8 six columns before the end, 1e-5 .. 1e-4 in the
    # last one), so they get 1e-3
    k = min(st.iters, so.iters)
    hg = gm.hessenberg(st.iters)
    off, dev = 0, []
    for j in range(1, k + 1):
        sl = slice(off, off + j + 1)
        off += j + 1
        dev.append(np.abs(hg[sl] - ho[sl]).max() / np.abs(ho[sl]).max())
    dev = np.array(dev)
    assert dev[:40].max() <= 1e-8, dev[:40].max()
    assert dev[:k - 6].max() <= 1e-6, (dev[:k - 6].max(), int(dev[:k - 6].argmax()))
    assert dev.max() <= 1e-3, (dev.max(), int(dev.argmax()))
    # true residual honours the tolerance
    r = b - P.jvp(u, x.to_host())
    assert np.linalg.norm(r) <= 1.05 * (1e-10 + 1e-10 * st.rnorm0) + 1e-9 * st.rnorm0


def test_gmres_restart_warmstart_operators(nls, ctx, po):
    N = 8
    dp, P, _ = make(nls, ctx, po, "bruss2d", N=N)
    u = P.u0()
    b = P.residual(u)
    J = P.dense_jac(u)
    xref = np.linalg.solve(J, b)
    # restarted GMRES(30)
    gm = nls.GmresSolver(ctx, P.n, nls.KrylovJL_GMRES(gmres_restart=30, itmax=5000), atol=0.0, rtol=1e-10)
    x, st = gm.solve(nls.JacobianOperator(dp, ctx.to_device(u)), ctx.to_device(b))
    xo, so = po.gmres(b, prob=P, u=u, opts=po.default_gmres_opts(atol=0.0, rtol=1e-10, restart=30, itmax=5000, orth=po.ORTH_CGS2))
    assert st.status == nls.abi.LS_SOLVED and st.restarts > 0 and abs(st.iters - so.iters) <= 30
    assert close(x.to_host(), xref, 1e-6)
    # warm start from a perturbed solution converges in fewer iterations to the same answer
    gm2 = nls.GmresSolver(ctx, P.n, nls.KrylovJL_GMRES(warm_start=True), atol=0.0, rtol=1e-10)
    x0 = ctx.to_device(xref * (1 + 1e-3))
    x2, st2 = gm2.solve(nls.JacobianOperator(dp, ctx.to_device(u)), ctx.to_device(b), x0)
    assert st2.status == nls.abi.LS_SOLVED and st2.nmatvec == st2.iters + 1 and close(x2.to_host(), xref, 1e-6)
    # dense and CSC operators (b2/b3 plug-in points)
    gm3 = nls.GmresSolver(ctx, P.n, nls.KrylovJL_GMRES(), atol=0.0, rtol=1e-10)
    x3, _ = gm3.solve(("dense", ctx.to_device(J.ravel(order="F"))), ctx.to_device(b))
    assert close(x3.to_host(), xref, 1e-6)
    cp, rv = P.pattern(1)
    col, nc = po.coloring_column(P.n, cp, rv)
    nz = P.sparse_jac(u, cp, rv, col, nc)
    x4, _ = gm3.solve(("csc", ctx.to_device(cp, np.int64), ctx.to_device(rv, np.int64), ctx.to_device(nz), 1), ctx.to_device(b))
    assert close(x4.to_host(), xref, 1e-6)
    # maxiters and zero right-hand side
    gm4 = nls.GmresSolver(ctx, P.n, nls.KrylovJL_GMRES(itmax=5), atol=0.0, rtol=1e-14)
    _, st4 = gm4.solve(nls.JacobianOperator(dp, ctx.to_device(u)), ctx.to_device(b))
    assert st4.status == nls.abi.LS_MAXITERS and st4.iters == 5
    x5, st5 = gm3.solve(nls.JacobianOperator(dp, ctx.to_device(u)), ctx.zeros(P.n))
    assert st5.status == nls.abi.LS_SOLVED and st5.iters == 0 and np.all(x5.to_host() == 0)


# ----------------------------------------------------------------------------- Newton (a4, a7, a8, a9)
def _cmp_newton(nls, po, sol, uo, ro, tro, exact_stats=True, trace_rtol=1e-6):
    assert sol.retcode == ro.retcode, (nls.ReturnCode.name(sol.retcode), ro.retcode)
    assert sol.stats.nsteps == ro.nsteps and sol.stats.nf == ro.nf
    if exact_stats:
        assert (sol.stats.njacs, sol.stats.nfactors, sol.stats.nsolve) == (ro.njacs, ro.nfactors, ro.nsolve)
    assert np.abs(sol.u - uo).max() <= RTOL_ROOT * np.abs(uo).max()
    assert abs(sol.resid_inf - np.abs(sol.resid).max()) <= 1e-300 + 1e-15 * sol.resid_inf
    for tg, t in zip(sol.trace, tro):
        assert tg.iter == t.iter
        if trace_rtol is not None:
            assert abs(tg.fnorm_inf - t.fnorm_inf) <= trace_rtol * max(t.fnorm_inf, 1e-9) + 1e-9


@pytest.mark.parametrize("variant", ["gmres", "gmres_mgs", "dense", "sparse", "tr", "ew", "fd"])
def test_newton_brusselator2d_vs_oracle(nls, ctx, po, golden, variant):
    # sparsity_tests__item1.jl:54-93 on the GPU: abstol = 1e-8 -> ||resid||_inf < 1e-8, and parity with the oracle run
    N = 32 if variant != "dense" else 16
    f = nls.Brusselator2D(N)
    P = po.OracleProblem.bruss2d(N)
    u0 = P.u0()
    kw = dict(abstol=1e-8)
    okw = dict(abstol=1e-8, gmres_orth=po.ORTH_CGS2)
    if variant == "gmres":
        alg = nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES())
    elif variant == "gmres_mgs":
        alg = nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(orth="mgs"))
        okw["gmres_orth"] = po.ORTH_MGS
    elif variant == "dense":
        alg = nls.NewtonRaphson()
        okw["linsolve"] = po.LINSOLVE_DENSE_LU
    elif variant == "sparse":
        alg = nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(), concrete_jac=True)
        okw["linsolve"] = po.LINSOLVE_SPARSE_GMRES
    elif variant == "tr":
        alg = nls.TrustRegion(linsolve=nls.KrylovJL_GMRES(), initial_trust_radius=10.0)
        okw.update(globalization=po.GLOB_TRUST_REGION, tr_initial_trust_radius=10.0)
    elif variant == "ew":
        alg = nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(), forcing=nls.EisenstatWalkerForcing2())
        okw["forcing"] = po.FORCING_EW2
    else:
        alg = nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(), jvp_autodiff=nls.AutoFiniteDiff())
        okw["jvp_mode"] = po.JVP_FINITE_DIFF
    sol = nls.solve(nls.NonlinearProblem(f, u0, (3.4, 1.0, 10.0), ctx=ctx), alg, **kw)
    uo, fo, ro, tro = P.newton(u0, po.default_newton_opts(**okw))
    assert np.abs(sol.resid).max() < 1e-8
    # finite-difference JVPs carry O(sqrt(eps)) noise that the inexact inner solves amplify along the way (not at the root)
    _cmp_newton(nls, po, sol, uo, ro, tro, trace_rtol=None if variant == "fd" else 1e-6)
    if N == 32:
        assert np.abs(sol.u - golden["root_32"]).max() <= RTOL_ROOT * np.abs(golden["root_32"]).max()
    if variant in ("gmres", "gmres_mgs", "sparse"):
        for tg, t in zip(sol.trace, tro):
            assert abs(tg.lin_iters - t.lin_iters) <= 2


def test_newton_quadratic_and_tridiag(nls, ctx, po, golden):
    # BASELINE config 1: f = u.^2 .- p, u0 = ones(1000), NewtonRaphson -> sqrt(2)  (rootfind_tests__item1.jl: err < 1e-9)
    for alg in (nls.NewtonRaphson(), nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES()), nls.TrustRegion(linsolve=nls.KrylovJL_GMRES())):
        sol = nls.solve(nls.NonlinearProblem(nls.QuadraticFunction(1000), np.ones(1000), 2.0, ctx=ctx), alg)
        assert nls.successful_retcode(sol.retcode)
        assert np.abs(sol.u - np.sqrt(2.0)).max() < 1e-9 and np.abs(sol.resid).max() < 1e-9
    assert sol.stats.nsteps >= 5
    # rootfind_tests__item20.jl:32-54 (custom jvp + GMRES, abstol 1e-13 -> < 1e-6), NewtonRaphson and TrustRegion
    p = golden["tridiag_p"]
    for alg in (nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES()), nls.TrustRegion(linsolve=nls.KrylovJL_GMRES())):
        sol = nls.solve(nls.NonlinearProblem(nls.TridiagQuadFunction(100), p, p, ctx=ctx), alg, abstol=1e-13)
        assert np.abs(sol.resid).max() < 1e-6
        assert np.abs(sol.u - golden["tridiag_root"]).max() < 1e-9


def test_newton_3d_vs_oracle(nls, ctx, po):
    N = 12
    P = po.OracleProblem.bruss3d(N)
    u0 = P.u0(1)
    sol = nls.solve(nls.NonlinearProblem(nls.Brusselator3D(N), u0, (3.4, 1.0, 10.0), ctx=ctx),
                    nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES()), abstol=1e-8)
    uo, fo, ro, tro = P.newton(u0, po.default_newton_opts(abstol=1e-8, gmres_orth=po.ORTH_CGS2))
    _cmp_newton(nls, po, sol, uo, ro, tro)
    # sparse concrete J + TrustRegion (BASELINE config 4 at test size)
    sol2 = nls.solve(nls.NonlinearProblem(nls.NonlinearFunction(nls.Brusselator3D(N), sparsity=nls.TracerSparsityDetector()), u0,
                                          (3.4, 1.0, 10.0), ctx=ctx), nls.TrustRegion(linsolve=nls.KrylovJL_GMRES()), abstol=1e-8)
    uo2, _, ro2, tro2 = P.newton(u0, po.default_newton_opts(abstol=1e-8, gmres_orth=po.ORTH_CGS2, linsolve=po.LINSOLVE_SPARSE_GMRES,
                                                            globalization=po.GLOB_TRUST_REGION))
    _cmp_newton(nls, po, sol2, uo2, ro2, tro2)


def test_iterator_interface_and_reinit(nls, ctx, po):
    # init / step! / solve! / reinit! (docs/src/tutorials/iterator_interface.md; solve.jl:108-133)
    N = 8
    P = po.OracleProblem.bruss2d(N)
    prob = nls.NonlinearProblem(nls.Brusselator2D(N), P.u0(), (3.4, 1.0, 10.0), ctx=ctx)
    cache = nls.init(prob, nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES()), abstol=1e-8)
    steps = 0
    while not nls.step_b(cache):
        steps += 1
        assert steps < 50
    sol = nls.solve_b(cache)
    assert sol.retcode == nls.ReturnCode.Success and sol.stats.nsteps == steps + 1
    nls.reinit_b(cache, P.u0() * 1.01)
    sol2 = nls.solve_b(cache)
    assert sol2.retcode == nls.ReturnCode.Success and np.abs(sol2.u - sol.u).max() < 1e-6 * np.abs(sol.u).max()
    # maxiters -> MaxIters (solve.jl:372-376)
    sol3 = nls.solve(prob, nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES()), abstol=1e-8, maxiters=1)
    assert sol3.retcode == nls.ReturnCode.MaxIters and sol3.stats.nsteps == 1
    # end-to-end host-buffer call
    cache2 = nls.init(prob, nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES()), abstol=1e-8)
    sol4 = cache2.solve_host(P.u0())
    assert np.abs(sol4.u - sol.u).max() < 1e-9 * np.abs(sol.u).max() and np.abs(sol4.resid).max() < 1e-8


def test_callback_problem_torch(nls, ctx, po, golden):
    # b1 plug-in point: NonlinearFunction{true}(F!; jvp = JVP!) with user closures running their own device code
    torch = pytest.importorskip("torch")
    p = torch.tensor(golden["tridiag_p"], device="cuda")
    n = p.numel()

    def T(x):
        y = 2.0 * x
        y[1:] -= x[:-1]
        y[:-1] -= x[1:]
        return y

    def F(du, u, _p):
        du_t, u_t = torch.as_tensor(du, device="cuda"), torch.as_tensor(u, device="cuda")
        du_t.copy_(u_t + 0.1 * u_t * T(u_t) - p)
        torch.cuda.synchronize()

    def JVP(Jv, v, u, _p):
        Jv_t, v_t, u_t = (torch.as_tensor(a, device="cuda") for a in (Jv, v, u))
        Jv_t.copy_(v_t + 0.1 * (u_t * T(v_t) + v_t * T(u_t)))
        torch.cuda.synchronize()

    for jvp in (JVP, None):  # None: the library falls back to the finite-difference JVP built from F alone
        prob = nls.NonlinearProblem(nls.NonlinearFunction(F, jvp=jvp, n=n), golden["tridiag_p"], None, ctx=ctx)
        sol = nls.solve(prob, nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES()), abstol=1e-12 if jvp else 1e-10)
        assert np.abs(sol.resid).max() < 1e-6
        assert np.abs(sol.u - golden["tridiag_root"]).max() < 1e-8


# ----------------------------------------------------------------------------- dense fallback (a5)
def test_dense_jacobian_and_lu(nls, ctx, po):
    N = 8
    dp, P, _ = make(nls, ctx, po, "bruss2d", N=N)
    u = P.u0() + 0.05
    J = dp.dense_jacobian(ctx.to_device(u)).to_host().reshape(P.n, P.n, order="F")
    assert close(J, P.dense_jac(u))
    d3, P3, _ = make(nls, ctx, po, "bruss3d", N=5)
    u3 = P3.u0(1)
    assert close(d3.dense_jacobian(ctx.to_device(u3)).to_host().reshape(P3.n, P3.n, order="F"), P3.dense_jac(u3))
    rng = np.random.default_rng(7)
    L = nls.abi.lib()
    for n in (1, 5, 31, 32, 33, 100, 257, 1000):
        A = rng.standard_normal((n, n))
        b = rng.standard_normal((n, 2))
        dA, dB = ctx.to_device(A.ravel(order="F")), ctx.to_device(b.ravel(order="F"))
        ipiv = ctx.empty(n, np.int64)
        info = C.c_int32(-1)
        nls.abi.check(ctx.handle, L.b200_getrf(ctx.handle, n, dA.ptr, n, ipiv.ptr, C.byref(info)))
        assert info.value == 0
        LUo, ipo, _ = po.getrf(A)
        assert np.array_equal(ipiv.to_host(), ipo)  # LAPACK pivot sequence, 1-based: bit-exact
        assert np.allclose(dA.to_host().reshape(n, n, order="F"), LUo, rtol=1e-9, atol=1e-11)
        nls.abi.check(ctx.handle, L.b200_getrs(ctx.handle, n, 2, dA.ptr, n, ipiv.ptr, dB.ptr, n))
        x = dB.to_host().reshape(n, 2, order="F")
        assert np.allclose(x, np.linalg.solve(A, b), rtol=1e-8, atol=1e-8)
    dZ = ctx.zeros(9)
    nls.abi.check(ctx.handle, L.b200_getrf(ctx.handle, 3, dZ.ptr, 3, ctx.empty(3, np.int64).ptr, C.byref(info)))
    assert info.value == 1


# ----------------------------------------------------------------------------- sparse fallback (a6)
@pytest.mark.parametrize("kind,N", [("bruss2d", 8), ("bruss2d", 32), ("bruss3d", 10)])
def test_sparse_pattern_coloring_fill(nls, ctx, po, golden, kind, N):
    dp, P, _ = make(nls, ctx, po, kind, N=N)
    for base in (0, 1):
        cp, rv = dp.pattern(base)
        cpo, rvo = P.pattern(base)
        assert np.array_equal(cp, cpo) and np.array_equal(rv, rvo)  # bit-exact index arrays
    if kind == "bruss2d":
        assert np.array_equal(cp, golden["colptr_%d" % N]) and np.array_equal(rv, golden["rowval_%d" % N])
    sj = nls.SparseJacobian(dp)
    co, nco = po.coloring_column(P.n, cpo, rvo, 1)
    assert sj.ncolors == nco and np.array_equal(sj.colors, co)  # bit-exact colour vector
    rng = np.random.default_rng(N)
    u = P.u0(1) + 0.1 * rng.standard_normal(P.n)
    nz = sj.fill(ctx.to_device(u))
    nzo = P.sparse_jac(u, cpo, rvo, co, nco)
    assert close(nz.to_host(), nzo)
    x = rng.standard_normal(P.n)
    assert close(sj.mul(nz, ctx.to_device(x)).to_host(), po.spmv(P.n, cpo, rvo, nzo, x))
    assert close(sj.mul(nz, ctx.to_device(x), transpose=True).to_host(), po.spmv(P.n, cpo, rvo, nzo, x, transpose=True))
    assert close(sj.mul(nz, ctx.to_device(x)).to_host(), P.jvp(u, x), 1e-11)
    # a user-supplied colorvec (ConstantColoringAlgorithm) is honoured
    sj2 = nls.SparseJacobian(dp, cp if base == 1 else None, rv if base == 1 else None, colors=co)
    assert close(sj2.fill(ctx.to_device(u)).to_host(), nzo)


# ----------------------------------------------------------------------------- ensemble (a11)
@pytest.mark.parametrize("N,K,orth", [(32, 40, "cgs2"), (32, 7, "mgs"), (16, 300, "cgs2"), (9, 5, "cgs2")])
def test_ensemble_batched_vs_oracle(nls, ctx, po, N, K, orth):
    # BASELINE config 5 at test size: the one-CTA-per-trajectory engine against per-trajectory oracle solves
    import bench
    P = po.OracleProblem.bruss2d(N)
    A, B = bench.ensemble_params(K)
    u0 = np.tile(P.u0(), (K, 1))
    u0 *= (1.0 + 0.01 * np.arange(K))[:, None]  # distinct initial conditions too
    alg = nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(orth=orth))
    cache = nls.EnsembleCache(ctx, N, K, 10.0, alg, abstol=1e-8)
    res = cache.solve(ctx.to_device(u0.ravel()), ctx.to_device(A), ctx.to_device(B))
    ocode = po.ORTH_MGS if orth == "mgs" else po.ORTH_CGS2
    uo, ro, rco, nso, njo, reso = po.ensemble_solve(N, u0, A, B, opts=po.default_newton_opts(abstol=1e-8, gmres_orth=ocode))
    u = cache.u_out.to_host().reshape(K, -1)
    assert res.nsuccess == K == reso.nsuccess
    assert np.array_equal(cache.rc.to_host(), rco) and np.array_equal(cache.ns.to_host(), nso)
    assert np.abs(u - uo).max() <= RTOL_ROOT * np.abs(uo).max()
    assert cache.resid.to_host().max() < 1e-8
    # iteration counts: same algorithm, reduction order differs -> each linear solve may stop at most 2 Arnoldi steps apart
    assert np.all(np.abs(cache.nj.to_host() - njo) <= 2 * nso), np.abs(cache.nj.to_host() - njo).max()
    # residual reported == residual of the returned iterate
    m = K // 2
    Pm = po.OracleProblem.bruss2d(N, A=A[m], B=B[m])
    assert abs(np.abs(Pm.residual(u[m])).max() - cache.resid.to_host()[m]) <= 1e-12 + 1e-6 * cache.resid.to_host()[m]


def test_ensemble_small(nls, ctx, po):
    N, K = 8, 6
    P = po.OracleProblem.bruss2d(N)
    prob = nls.NonlinearProblem(nls.Brusselator2D(N), P.u0(), (3.4, 1.0, 10.0), ctx=ctx)
    pf = lambda pr, i, rep: nls.remake(pr, p=(3.4 + 0.1 * ((i - 1) % 64) / 64, 1.0 + 0.05 * ((i - 1) // 2) / 128, 10.0))  # noqa: E731
    es = nls.solve(nls.EnsembleProblem(prob, prob_func=pf), nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES()), nls.EnsembleB200(),
                   trajectories=K, abstol=1e-8)
    A = np.array([3.4 + 0.1 * (m % 64) / 64 for m in range(K)])
    B = np.array([1.0 + 0.05 * (m // 2) / 128 for m in range(K)])
    uo, ro, rco, nso, njo, reso = po.ensemble_solve(N, np.tile(P.u0(), (K, 1)), A, B, opts=po.default_newton_opts(abstol=1e-8, gmres_orth=po.ORTH_CGS2))
    assert es.converged() and es.summary.nsuccess == K  # core_tests__item6.jl:14-20
    assert np.array_equal(es.retcodes, rco) and np.array_equal(es.nsteps, nso)
    assert np.abs(es.u - uo).max() <= RTOL_ROOT * np.abs(uo).max()
    assert es.resid_inf.max() < 1e-8
