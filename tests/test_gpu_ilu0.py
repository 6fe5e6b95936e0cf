"""ILU(0) on the device (csrc/ilu0.cu, b200_ilu0_*) and as the `precs` of GMRES on the sparse route.

Exact probes: an integer unit-lower L and an integer U whose diagonal is +-powers of two give A = L U exactly; on the pattern
struct(L U) every intermediate of the factorisation and of the two sweeps is an exact integer, so the factors and the solve
must come back bit for bit.  The Brusselator Jacobians are checked against the NumPy restatement (oracle/ilu0_numpy.py)."""
import numpy as np
import pytest
import scipy.sparse as sp

from oracle import ilu0_numpy as il

pytestmark = pytest.mark.gpu


def _csc_of(S, A, index_base):
    """CSC (colptr, rowval, nzval) of the structure S with the values of A (dense arrays; small cases)."""
    n = S.shape[0]
    colptr, rowval, nzval = [0], [], []
    for c in range(n):
        r = np.nonzero(S[:, c])[0]
        rowval.extend(r.tolist())
        nzval.extend(A[r, c].tolist())
        colptr.append(len(rowval))
    return np.array(colptr, dtype=np.int64) + index_base, np.array(rowval, dtype=np.int64) + index_base, np.array(nzval, dtype=np.float64)


def _probe(kind, n, seed):
    """Integer factors as sparse int64 matrices: L unit lower, U upper with a +-power-of-two diagonal."""
    rng = np.random.default_rng(seed)
    li, lj, lv, ui, uj, uv = [], [], [], [], [], []
    if kind == "random":
        plain = set(rng.choice(n, size=n // 4, replace=False).tolist())   # rows (and columns) with nothing but the diagonal
        for i in range(n):
            for j in rng.choice(n, size=min(n, 3), replace=False).tolist():
                if i in plain or j in plain or i == j:
                    continue
                for lst, v in zip((li, lj, lv) if j < i else (ui, uj, uv), (i, j, int(rng.choice([-2, -1, 1, 2])))):
                    lst.append(v)
    elif kind == "chain":            # tridiagonal A: n levels in each sweep
        idx = np.arange(1, n)
        li, lj, lv = idx, idx - 1, rng.choice([-1, 1], n - 1)
        ui, uj, uv = idx - 1, idx, rng.choice([-1, 1], n - 1)
    elif kind == "arrow":            # last row and last column full: a row of n > 32 entries
        idx = np.arange(n - 1)
        li, lj, lv = np.full(n - 1, n - 1), idx, rng.choice([-1, 1], n - 1)
        ui, uj, uv = idx, np.full(n - 1, n - 1), rng.choice([-1, 1], n - 1)
    # kind == "diagonal": one level
    d = rng.choice([-4, -2, -1, 1, 2, 4], n)
    L = sp.csr_matrix((np.concatenate([np.ones(n), lv]).astype(np.int64), (np.concatenate([np.arange(n), li]), np.concatenate([np.arange(n), lj]))), shape=(n, n))
    U = sp.csr_matrix((np.concatenate([d, uv]).astype(np.int64), (np.concatenate([np.arange(n), ui]), np.concatenate([np.arange(n), uj]))), shape=(n, n))
    return L, U


def _exact_case(kind, n, base, seed=0):
    L, U = _probe(kind, n, seed)
    A = (L @ U).tocsc()                                          # exact in int64
    S = (abs(L) @ abs(U)).tocsc()                                # struct(L U): no cancellation, explicit zeros of A kept
    S.sort_indices()
    colptr = S.indptr.astype(np.int64) + base
    rows = S.indices.astype(np.int64)
    cols = np.repeat(np.arange(n), np.diff(S.indptr))
    nz = np.asarray(A[rows, cols]).ravel().astype(np.float64)
    packed = np.where(rows > cols, np.asarray(L[rows, cols]).ravel(), np.asarray(U[rows, cols]).ravel()).astype(np.float64)
    return colptr, rows + base, nz, packed, A


PROBES = [("random", 1, 1), ("random", 31, 0), ("random", 32, 1), ("random", 33, 0), ("random", 257, 1), ("chain", 20000, 0),
          ("chain", 20000, 1), ("diagonal", 1000, 1), ("arrow", 40, 0), ("arrow", 257, 1)]


@pytest.mark.parametrize("kind,n,base", PROBES)
def test_exact_probes_bit_for_bit(nls, ctx, kind, n, base):
    colptr, rowval, nz, packed, A = _exact_case(kind, n, base, seed=n + base)
    ilu = nls.SparseILU0(ctx, n, colptr, rowval, base)
    lo, up = ilu.levels()
    assert (lo, up) == il.level_counts(n, colptr, rowval, base)
    if kind == "chain":
        assert lo == up == n
    if kind == "diagonal":
        assert lo == up == 1
    assert ilu.factor(ctx.to_device(nz)) == 0
    assert np.array_equal(ilu.factors().to_host(), packed)
    xt = np.random.default_rng(n).integers(-3, 4, n).astype(np.float64)
    b = (A @ xt.astype(np.int64)).astype(np.float64)          # exact: A and xt are small integers
    assert np.array_equal(ilu.solve(ctx.to_device(b)).to_host(), xt)
    db = ctx.to_device(b)                                      # x may alias b
    ilu.solve(db, db)
    assert np.array_equal(db.to_host(), xt)


def _bruss_case(nls, ctx, dim, N):
    f = nls.Brusselator2D(N) if dim == 2 else nls.Brusselator3D(N)
    dp = nls._DeviceProblem(ctx, nls.NonlinearProblem(f, None, (3.4, 1.0, 10.0), ctx=ctx))
    u = dp.u0(nls.abi.U0_PERTURBED_Z)
    sj = nls.SparseJacobian(dp)
    nz = sj.fill(u)
    return dp, u, sj, nz


@pytest.mark.parametrize("dim,N", [(2, 32), (3, 16)])
def test_brusselator_against_the_restatement(nls, ctx, dim, N):
    dp, u, sj, nz = _bruss_case(nls, ctx, dim, N)
    n = dp.n
    ilu = nls.SparseILU0(ctx, n, sj.colptr, sj.rowval, 1)
    assert ilu.levels() == il.level_counts(n, sj.colptr, sj.rowval, 1) == ((2 * N, 2 * N) if dim == 2 else (3 * N - 1, 3 * N - 1))
    nzh = nz.to_host()
    fo, info = il.ilu0(n, sj.colptr, sj.rowval, nzh, 1)
    assert info == 0 and ilu.factor(nz) == 0
    f1 = ilu.factors().to_host()
    assert np.abs(f1 - fo).max() <= 1e-13 * np.abs(fo).max()
    b = np.random.default_rng(dim).standard_normal(n)
    xo = il.solve(n, sj.colptr, sj.rowval, fo, b, 1)
    x1 = ilu.solve(ctx.to_device(b)).to_host()
    assert np.abs(x1 - xo).max() <= 1e-13 * np.abs(xo).max()
    # bit-reproducible: a second factorisation and a second solve
    assert ilu.factor(nz) == 0
    assert np.array_equal(ilu.factors().to_host(), f1)
    assert np.array_equal(ilu.solve(ctx.to_device(b)).to_host(), x1)


def test_error_paths(nls, ctx):
    # a row without a structural diagonal: create fails and names the row (1-based pattern: row 3 holds only column 1)
    colptr = np.array([1, 3, 4, 5], dtype=np.int64)
    rowval = np.array([1, 3, 2, 1], dtype=np.int64)
    with pytest.raises(nls.abi.B200Error) as e:
        nls.SparseILU0(ctx, 3, colptr, rowval, 1)
    assert e.value.code == nls.abi.ERR_INVALID and "row 3" in str(e.value)
    # zero pivots: u_22 = 1 - 1 * 1 = 0 and a zero at row 5; the first row is reported (1-based)
    n = 6
    A = np.eye(n)
    A[0, 1] = A[1, 0] = 1.0
    A[4, 4] = 0.0
    S = (A != 0) | np.eye(n, dtype=bool)
    colptr, rowval, nz = _csc_of(S, A, 1)
    ilu = nls.SparseILU0(ctx, n, colptr, rowval, 1)
    assert ilu.factor(ctx.to_device(nz)) == 2
    A[0, 1] = 0.5
    colptr, rowval, nz = _csc_of(S, A, 1)
    assert ilu.factor(ctx.to_device(nz)) == 5


def test_newton_refuses_ilu0_where_it_cannot_run(nls, ctx):
    N = 8
    f = nls.Brusselator2D(N)
    u0 = nls._DeviceProblem(ctx, nls.NonlinearProblem(f, None, (3.4, 1.0, 10.0), ctx=ctx)).u0(nls.abi.U0_PERTURBED_Z).to_host()
    prob = nls.NonlinearProblem(f, u0, (3.4, 1.0, 10.0), ctx=ctx)
    with pytest.raises(nls.abi.B200Error) as e:   # matrix-free GMRES: there is no assembled matrix to factor
        nls.solve(prob, nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(precs=nls.ILU0("left"))), abstol=1e-8)
    assert e.value.code == nls.abi.ERR_INVALID and "concrete_jac = true" in str(e.value)
    with pytest.raises(nls.abi.B200Error) as e:   # the SER shift would need a refactorisation every step
        nls.solve(prob, nls.PseudoTransient(concrete_jac=True, linsolve=nls.KrylovJL_GMRES(precs=nls.ILU0("left"))), abstol=1e-8)
    assert e.value.code == nls.abi.ERR_UNSUPPORTED and "PseudoTransient" in str(e.value)


# Left preconditioning makes GMRES test the PRECONDITIONED residual (~1/diag(J) times the true one), so the inherited absolute
# tolerance would stop the linear solves far too early; a left-preconditioned run sets the Krylov tolerances itself, as
# tests/test_precond.py does for block-Jacobi.
def _krylov_kw(side):
    return dict(atol=1e-13, rtol=1e-9) if side == "left" else {}


def _iters_per_step(sol):
    return sum(t.lin_iters for t in sol.trace) / max(1, len(sol.trace))


def _compare(nls, sol0, sol1):
    assert sol0.retcode == sol1.retcode == nls.ReturnCode.Success
    assert np.abs(sol1.u - sol0.u).max() <= 1e-6 * np.abs(sol0.u).max()
    assert _iters_per_step(sol1) < _iters_per_step(sol0)
    assert sol1.stats.nfactors == sol0.stats.nfactors == 0      # the preconditioner build is not an NLStats factorisation


@pytest.mark.parametrize("side", ["left", "right"])
def test_newton_raphson_2d_with_ilu0(nls, ctx, side):
    N = 32
    f = nls.Brusselator2D(N)
    u0 = nls._DeviceProblem(ctx, nls.NonlinearProblem(f, None, (3.4, 1.0, 10.0), ctx=ctx)).u0(nls.abi.U0_PERTURBED_Z).to_host()
    prob = nls.NonlinearProblem(f, u0, (3.4, 1.0, 10.0), ctx=ctx)
    s0 = nls.solve(prob, nls.NewtonRaphson(concrete_jac=True, linsolve=nls.KrylovJL_GMRES()), abstol=1e-8)
    s1 = nls.solve(prob, nls.NewtonRaphson(concrete_jac=True, linsolve=nls.KrylovJL_GMRES(precs=nls.ILU0(side), **_krylov_kw(side))), abstol=1e-8)
    _compare(nls, s0, s1)


@pytest.mark.parametrize("side", ["left", "right"])
def test_trust_region_3d_with_ilu0(nls, ctx, side):
    N = 16
    f = nls.Brusselator3D(N)
    u0 = nls._DeviceProblem(ctx, nls.NonlinearProblem(f, None, (3.4, 1.0, 10.0), ctx=ctx)).u0(nls.abi.U0_PERTURBED_Z).to_host()
    fs = nls.NonlinearFunction(f, sparsity=nls.TracerSparsityDetector())
    prob = nls.NonlinearProblem(fs, u0, (3.4, 1.0, 10.0), ctx=ctx)
    s0 = nls.solve(prob, nls.TrustRegion(linsolve=nls.KrylovJL_GMRES(orth="mgs")), abstol=1e-8)
    s1 = nls.solve(prob, nls.TrustRegion(linsolve=nls.KrylovJL_GMRES(orth="mgs", precs=nls.ILU0(side), **_krylov_kw(side))), abstol=1e-8)
    _compare(nls, s0, s1)


def test_left_preconditioned_gmres_matches_the_oracle(nls, ctx, po):
    """One left-preconditioned GMRES solve on the assembled 2D N = 32 Jacobian against the oracle's GMRES on the explicit
    dense operator (M^-1 J, M^-1 b), M = L U of the restatement."""
    dp, u, sj, nz = _bruss_case(nls, ctx, 2, 32)
    n = dp.n
    nzh = nz.to_host()
    fo, _ = il.ilu0(n, sj.colptr, sj.rowval, nzh, 1)
    Lo, Uo = il.dense_factors(n, sj.colptr, sj.rowval, fo, 1)
    J = np.zeros((n, n))
    cols = np.repeat(np.arange(n), np.diff(sj.colptr))
    J[sj.rowval - 1, cols] = nzh
    b = dp.residual(u).to_host()
    Minv_J = np.linalg.solve(Uo, np.linalg.solve(Lo, J))
    Minv_b = np.linalg.solve(Uo, np.linalg.solve(Lo, b))
    opts = po.default_gmres_opts(atol=1e-10, rtol=1e-10, orth=po.ORTH_CGS2)
    xo, so = po.gmres(Minv_b, dense=Minv_J, opts=opts)
    ilu = nls.SparseILU0(ctx, n, sj.colptr, sj.rowval, 1)
    assert ilu.factor(nz) == 0
    gm = nls.GmresSolver(ctx, n, nls.KrylovJL_GMRES(orth="cgs2"), atol=1e-10, rtol=1e-10)
    x, st = gm.solve(("sparse_jac", sj, nz), ctx.to_device(b), Pl=ilu.linop())
    assert st.status == nls.abi.LS_SOLVED == so.status and abs(st.iters - so.iters) <= 1
    assert abs(st.rnorm0 - so.rnorm0) <= 1e-10 * so.rnorm0        # the stopping test sees the preconditioned residual
    assert np.abs(x.to_host() - xo).max() <= 1e-7 * np.abs(xo).max()
    gm0 = nls.GmresSolver(ctx, n, nls.KrylovJL_GMRES(orth="cgs2"), atol=1e-10, rtol=1e-10)
    _, st0 = gm0.solve(("sparse_jac", sj, nz), ctx.to_device(b))
    assert st.iters < st0.iters


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
def test_user_callback_with_jac_prototype_and_ilu0(nls, ctx, side):
    fn, u0 = _user_reaction_diffusion(nls, ctx, 32)
    prob = nls.NonlinearProblem(fn, u0, None, ctx=ctx)
    s0 = nls.solve(prob, nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES()), abstol=1e-9)
    s1 = nls.solve(prob, nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(precs=nls.ILU0(side), **_krylov_kw(side))), abstol=1e-9)
    _compare(nls, s0, s1)
    assert np.abs(s1.u - 1.0).max() < 1e-8                      # the root is u = 1
