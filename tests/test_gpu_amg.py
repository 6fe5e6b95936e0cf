"""Ruge-Stueben AMG on the device (csrc/amg.cu, b200_amg_*) and as the `precs` of GMRES on the sparse route.

The device hierarchy is checked against the NumPy restatement (oracle/amg_numpy.py): level sizes, splittings and every pattern
exactly, values and one V-cycle to rounding; refreshes and applications bit for bit against themselves."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import amg_numpy as am

pytestmark = pytest.mark.gpu


def _bruss_case(nls, ctx, dim, N):
    f = nls.Brusselator2D(N) if dim == 2 else nls.Brusselator3D(N)
    dp = nls._DeviceProblem(ctx, nls.NonlinearProblem(f, None, (3.4, 1.0, 10.0), ctx=ctx))
    u = dp.u0(nls.abi.U0_PERTURBED_Z)
    sj = nls.SparseJacobian(dp)
    nz = sj.fill(u)
    return dp, u, sj, nz


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def _same_as_restatement(amg, H):
    ns, nzs = amg.levels()
    assert ns == H.sizes() and nzs == H.nnz()
    for l in range(len(ns)):
        lv = amg.level(l)
        Ao = H.levels[l]["A"] if l < len(H.levels) else H.coarse
        val, col, rowptr = lv["A"]
        assert np.array_equal(rowptr, Ao.indptr) and np.array_equal(col, Ao.indices)
        assert _rel(val, Ao.data) <= 1e-13
        if l < len(H.levels):
            Po = H.levels[l]["P"]
            val, col, rowptr = lv["P"]
            assert np.array_equal(rowptr, Po.indptr) and np.array_equal(col, Po.indices)   # the splitting: C rows are unit rows
            assert _rel(val, Po.data) <= 1e-13
        else:
            assert lv["P"] is None


def _snapshot(amg):
    out = []
    for l in range(len(amg.levels()[0])):
        lv = amg.level(l)
        out.append([a.copy() for M in (lv["A"], lv["P"]) if M is not None for a in M])
    return out


def _bits_equal(s1, s2):
    return all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for x, y in zip(s1, s2) for a, b in zip(x, y)) and len(s1) == len(s2)


@pytest.mark.parametrize("dim,N", [(2, 32), (3, 16)])
def test_hierarchy_against_the_restatement(nls, ctx, dim, N):
    dp, u, sj, nz = _bruss_case(nls, ctx, dim, N)
    n = dp.n
    amg = nls.SparseAMG(ctx, n, sj.colptr, sj.rowval, 1)
    assert amg.setup(nz) == 0
    H = am.Hierarchy(am.csr_of_csc(n, sj.colptr, sj.rowval, nz.to_host(), 1))
    if dim == 2:
        assert H.sizes() == [2048, 1024, 256, 64, 16, 4]
    _same_as_restatement(amg, H)
    rng = np.random.default_rng(dim)
    for _ in range(3):
        b = rng.standard_normal(n)
        x = amg.solve(ctx.to_device(b)).to_host()
        assert _rel(x, H.cycle(b)) <= 1e-12
    # bit-reproducible applications; x may alias b
    db = ctx.to_device(b)
    x1 = amg.solve(db).to_host()
    assert np.array_equal(x1, amg.solve(db).to_host())
    amg.solve(db, db)
    assert np.array_equal(db.to_host(), x1)


@pytest.mark.parametrize("dim,N", [(2, 32), (3, 16)])
def test_refresh_keeps_the_splitting_and_is_bit_reproducible(nls, ctx, dim, N):
    dp, u, sj, nz = _bruss_case(nls, ctx, dim, N)
    n = dp.n
    amg = nls.SparseAMG(ctx, n, sj.colptr, sj.rowval, 1)
    assert amg.setup(nz, rebuild=True) == 0
    rebuilt = _snapshot(amg)
    b = ctx.to_device(np.random.default_rng(7).standard_normal(n))
    x_rebuilt = amg.solve(b).to_host()
    H = am.Hierarchy(am.csr_of_csc(n, sj.colptr, sj.rowval, nz.to_host(), 1))
    # new values: the Jacobian at another state, on the frozen splitting
    u2 = ctx.to_device(u.to_host() * (1.0 + 0.05 * np.sin(np.arange(n))))
    nz2 = sj.fill(u2)
    assert amg.setup(nz2, rebuild=False) == 0
    H2 = H.refresh(am.csr_of_csc(n, sj.colptr, sj.rowval, nz2.to_host(), 1))
    _same_as_restatement(amg, H2)
    bh = b.to_host()
    assert _rel(amg.solve(b).to_host(), H2.cycle(bh)) <= 1e-12
    s2 = _snapshot(amg)
    assert amg.setup(nz2, rebuild=False) == 0            # two refreshes at the same values
    assert _bits_equal(s2, _snapshot(amg))
    assert amg.setup(nz, rebuild=False) == 0             # a refresh and a rebuild at the same values
    assert _bits_equal(rebuilt, _snapshot(amg))
    assert np.array_equal(amg.solve(b).to_host(), x_rebuilt)


def _csc_of(A, base=1):
    A = sp.csc_matrix(A)
    A.sort_indices()
    return A.indptr.astype(np.int64) + base, A.indices.astype(np.int64) + base, A.data.astype(np.float64)


def test_error_paths(nls, ctx):
    # a row without a structural diagonal: create fails and names the row (row 3 holds only column 1)
    colptr = np.array([1, 3, 4, 5], dtype=np.int64)
    rowval = np.array([1, 3, 2, 1], dtype=np.int64)
    with pytest.raises(nls.abi.B200Error) as e:
        nls.SparseAMG(ctx, 3, colptr, rowval, 1)
    assert e.value.code == nls.abi.ERR_INVALID and "row 3" in str(e.value)
    # a zero (stored) diagonal on the finest level: info names level 1
    n = 40
    A = 2.0 * np.eye(n) - np.eye(n, k=1) - np.eye(n, k=-1)
    S = A != 0
    A[17, 17] = 0.0
    cp, rv, _ = _csc_of(S.astype(np.float64))
    nzv = A[rv - 1, np.repeat(np.arange(n), np.diff(cp))]
    amg = nls.SparseAMG(ctx, n, cp, rv, 1)
    assert amg.setup(ctx.to_device(nzv)) == 1
    # a hierarchy ending above the dense cap
    dp, u, sj, nz = _bruss_case(nls, ctx, 2, 64)
    amg = nls.SparseAMG(ctx, dp.n, sj.colptr, sj.rowval, 1, max_levels=1)
    with pytest.raises(nls.abi.B200Error) as e:
        amg.setup(nz)
    assert e.value.code == nls.abi.ERR_UNSUPPORTED and "8192" in str(e.value) and "raise max_levels" in str(e.value)
    # a refresh needs a hierarchy
    amg = nls.SparseAMG(ctx, dp.n, sj.colptr, sj.rowval, 1)
    with pytest.raises(nls.abi.B200Error):
        amg.setup(nz, rebuild=False)


def test_newton_refuses_amg_where_it_cannot_run(nls, ctx):
    N = 8
    f = nls.Brusselator2D(N)
    dp = nls._DeviceProblem(ctx, nls.NonlinearProblem(f, None, (3.4, 1.0, 10.0), ctx=ctx))
    u0 = dp.u0(nls.abi.U0_PERTURBED_Z).to_host()
    prob = nls.NonlinearProblem(f, u0, (3.4, 1.0, 10.0), ctx=ctx)
    with pytest.raises(nls.abi.B200Error) as e:   # matrix-free GMRES: there is no assembled matrix to coarsen
        nls.solve(prob, nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(precs=nls.RugeStubenAMG("left"))), abstol=1e-8)
    assert e.value.code == nls.abi.ERR_INVALID and "concrete_jac = true" in str(e.value)
    with pytest.raises(nls.abi.B200Error) as e:
        nls.solve(prob, nls.PseudoTransient(concrete_jac=True, linsolve=nls.KrylovJL_GMRES(precs=nls.RugeStubenAMG("right"))), abstol=1e-8)
    assert e.value.code == nls.abi.ERR_UNSUPPORTED and "PseudoTransient" in str(e.value)
    L = nls.abi.lib()
    for linsolve in (nls.abi.LINSOLVE_DENSE_LU, nls.abi.LINSOLVE_SPARSE_LU):   # no Krylov method to precondition
        o = nls.abi.NewtonOpts()
        L.b200_newton_opts_default(C.byref(o))
        o.linsolve, o.precond = linsolve, nls.abi.PRECOND_AMG_LEFT
        h = C.c_void_p()
        assert L.b200_newton_create(dp.handle, C.byref(o), C.byref(h)) == nls.abi.ERR_INVALID
        assert "concrete_jac = true" in L.b200_last_error(ctx.handle).decode()


# Left preconditioning makes GMRES test the preconditioned residual, so a left-preconditioned run sets the Krylov tolerances
# itself, as the ILU(0) tests do (DESIGN.md §4g)
def _krylov_kw(side):
    return dict(atol=1e-13, rtol=1e-9) if side == "left" else {}


def _iters_per_step(sol):
    return sum(t.lin_iters for t in sol.trace) / max(1, len(sol.trace))


def _compare(nls, sol0, sol1):
    assert sol0.retcode == sol1.retcode == nls.ReturnCode.Success
    assert np.abs(sol1.u - sol0.u).max() <= 1e-8 * max(1.0, np.abs(sol0.u).max())
    assert _iters_per_step(sol1) < _iters_per_step(sol0)
    assert sol1.stats.nfactors == sol0.stats.nfactors == 0      # the hierarchy is not an NLStats factorisation


@pytest.mark.parametrize("side", ["left", "right"])
def test_newton_raphson_2d_with_amg(nls, ctx, side):
    N = 32
    f = nls.Brusselator2D(N)
    u0 = nls._DeviceProblem(ctx, nls.NonlinearProblem(f, None, (3.4, 1.0, 10.0), ctx=ctx)).u0(nls.abi.U0_PERTURBED_Z).to_host()
    prob = nls.NonlinearProblem(f, u0, (3.4, 1.0, 10.0), ctx=ctx)
    s0 = nls.solve(prob, nls.NewtonRaphson(concrete_jac=True, linsolve=nls.KrylovJL_GMRES()), abstol=1e-8)
    s1 = nls.solve(prob, nls.NewtonRaphson(concrete_jac=True, linsolve=nls.KrylovJL_GMRES(precs=nls.RugeStubenAMG(side), **_krylov_kw(side))), abstol=1e-8)
    _compare(nls, s0, s1)


@pytest.mark.parametrize("side", ["left", "right"])
def test_trust_region_3d_with_amg(nls, ctx, side):
    N = 16
    f = nls.Brusselator3D(N)
    u0 = nls._DeviceProblem(ctx, nls.NonlinearProblem(f, None, (3.4, 1.0, 10.0), ctx=ctx)).u0(nls.abi.U0_PERTURBED_Z).to_host()
    fs = nls.NonlinearFunction(f, sparsity=nls.TracerSparsityDetector())
    prob = nls.NonlinearProblem(fs, u0, (3.4, 1.0, 10.0), ctx=ctx)
    s0 = nls.solve(prob, nls.TrustRegion(linsolve=nls.KrylovJL_GMRES(orth="mgs")), abstol=1e-8)
    s1 = nls.solve(prob, nls.TrustRegion(linsolve=nls.KrylovJL_GMRES(orth="mgs", precs=nls.RugeStubenAMG(side), **_krylov_kw(side))), abstol=1e-8)
    _compare(nls, s0, s1)


def _user_reaction_diffusion(nls, ctx, N):
    """A user residual on the GPU (torch): periodic 5-point diffusion with a cubic reaction, F(u) = a (4u - sum of the four
    neighbours) + u^3 - 1 on an N x N grid, with its 5-point jac_prototype (1-based CSC) and no jac!."""
    torch = pytest.importorskip("torch")
    n = N * N
    a = 0.25 * N * N

    def lap(x):
        g = x.view(N, N)
        return (4.0 * g - g.roll(1, 0) - g.roll(-1, 0) - g.roll(1, 1) - g.roll(-1, 1)).reshape(-1)

    def F(du, u, _p):
        du_t, u_t = torch.as_tensor(du, device="cuda"), torch.as_tensor(u, device="cuda")
        du_t.copy_(a * lap(u_t) + u_t ** 3 - 1.0)
        torch.cuda.synchronize()

    def JVP(Jv, v, u, _p):
        Jv_t, v_t, u_t = (torch.as_tensor(x, device="cuda") for x in (Jv, v, u))
        Jv_t.copy_(a * lap(v_t) + 3.0 * u_t * u_t * v_t)
        torch.cuda.synchronize()

    colptr, rowval = [1], []
    for c in range(n):
        i, j = c % N, c // N
        rs = sorted({c, (i + 1) % N + N * j, (i - 1) % N + N * j, i + N * ((j + 1) % N), i + N * ((j - 1) % N)})
        rowval.extend(r + 1 for r in rs)
        colptr.append(len(rowval) + 1)
    proto = (np.array(colptr, dtype=np.int64), np.array(rowval, dtype=np.int64), 1)
    u0 = 0.5 + 0.1 * np.sin(np.arange(n))
    return nls.NonlinearFunction(F, jvp=JVP, n=n, jac_prototype=proto), u0


@pytest.mark.parametrize("side", ["left", "right"])
def test_user_callback_with_jac_prototype_and_amg(nls, ctx, side):
    fn, u0 = _user_reaction_diffusion(nls, ctx, 32)
    prob = nls.NonlinearProblem(fn, u0, None, ctx=ctx)
    s0 = nls.solve(prob, nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES()), abstol=1e-9)
    s1 = nls.solve(prob, nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(precs=nls.RugeStubenAMG(side), **_krylov_kw(side))), abstol=1e-9)
    _compare(nls, s0, s1)
    assert np.abs(s1.u - 1.0).max() < 1e-8                      # the root is u = 1
