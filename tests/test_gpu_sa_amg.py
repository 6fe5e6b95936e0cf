"""Smoothed-aggregation AMG on the device (csrc/amg.cu, b200_amg_create_sa) and as the `precs` of GMRES on the sparse route.

The device hierarchy is checked against the NumPy restatement (oracle/sa_numpy.py): level sizes, every tentative prolongator
(the aggregates) and every pattern of A and P exactly, values and one V-cycle to rounding; rebuilds and refreshes bit for bit
against each other; at config-4 size, A_c = P' A P on every level and MIS-2 on level 0."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import sa_numpy as sa
from test_amg_oracle import graph_laplacian, random_matrix
from test_gpu_amg import _bits_equal, _bruss_case, _csc_of, _iters_per_step, _krylov_kw, _rel, _user_reaction_diffusion

pytestmark = pytest.mark.gpu


def _csr(M):
    val, col, rowptr = M
    return sp.csr_matrix((val, col, rowptr), shape=(len(rowptr) - 1, len(rowptr) - 1))


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
            for key in ("T", "P"):
                Mo = H.levels[l][key]
                val, col, rowptr = lv[key]
                assert np.array_equal(rowptr, Mo.indptr) and np.array_equal(col, Mo.indices), key
                assert _rel(val, Mo.data) <= 1e-13, key
        else:
            assert lv["P"] is None and lv["T"] is None


def _snapshot(amg):
    out = []
    for l in range(len(amg.levels()[0])):
        lv = amg.level(l)
        out.append([a.copy() for k in ("A", "P", "T") if lv[k] is not None for a in lv[k]])
    return out


def _matrix_case(ctx, A):
    A = sp.csr_matrix(A)
    cp, rv, nz = _csc_of(A)
    return A.shape[0], cp, rv, nz, ctx.to_device(nz)


def _cases(nls, ctx):
    out = []
    for dim, N in ((2, 32), (3, 16)):
        dp, u, sj, nz = _bruss_case(nls, ctx, dim, N)
        out.append(("bruss%dd" % dim, dp.n, sj.colptr, sj.rowval, nz.to_host(), nz))
    for name, A in (("random", random_matrix(3000, 5)), ("laplacian", graph_laplacian(3000, 2) + 0.1 * sp.identity(3000))):
        n, cp, rv, nzh, nzd = _matrix_case(ctx, A)
        out.append((name, n, cp, rv, nzh, nzd))
    return out


def test_hierarchy_against_the_restatement(nls, ctx):
    for name, n, cp, rv, nzh, nzd in _cases(nls, ctx):
        amg = nls.SparseAMG.smoothed_aggregation(ctx, n, cp, rv, 1)
        assert amg.setup(nzd) == 0, name
        H = sa.Hierarchy(sa.am.csr_of_csc(n, cp, rv, nzh, 1))
        assert len(H.sizes()) >= 2, name
        if name == "laplacian":
            assert (H.levels[0]["agg"] < 0).any()           # isolated rows: empty rows of T
        _same_as_restatement(amg, H)
        b = np.random.default_rng(1).standard_normal(n)
        assert _rel(amg.solve(ctx.to_device(b)).to_host(), H.cycle(b)) <= 1e-12, name


@pytest.mark.parametrize("dim,N", [(2, 32), (3, 16)])
def test_rebuild_and_refresh_bits(nls, ctx, dim, N):
    dp, u, sj, nz = _bruss_case(nls, ctx, dim, N)
    n = dp.n
    amg = nls.SparseAMG.smoothed_aggregation(ctx, n, sj.colptr, sj.rowval, 1)
    assert amg.setup(nz) == 0
    first = _snapshot(amg)
    b = ctx.to_device(np.random.default_rng(7).standard_normal(n))
    x_first = amg.solve(b).to_host()
    assert amg.setup(nz) == 0                             # two rebuilds at the same values
    assert _bits_equal(first, _snapshot(amg))
    assert np.array_equal(amg.solve(b).to_host(), x_first)
    H = sa.Hierarchy(sa.am.csr_of_csc(n, sj.colptr, sj.rowval, nz.to_host(), 1))
    u2 = ctx.to_device(u.to_host() * (1.0 + 0.05 * np.sin(np.arange(n))))
    nz2 = sj.fill(u2)
    assert amg.setup(nz2, rebuild=False) == 0             # new values on the frozen aggregates
    H2 = H.refresh(sa.am.csr_of_csc(n, sj.colptr, sj.rowval, nz2.to_host(), 1))
    _same_as_restatement(amg, H2)
    assert _rel(amg.solve(b).to_host(), H2.cycle(b.to_host())) <= 1e-12
    s2 = _snapshot(amg)
    assert amg.setup(nz2, rebuild=False) == 0
    assert _bits_equal(s2, _snapshot(amg))
    assert amg.setup(nz, rebuild=False) == 0              # a refresh and a rebuild at the same values
    assert _bits_equal(first, _snapshot(amg))
    assert np.array_equal(amg.solve(b).to_host(), x_first)


def test_error_paths(nls, ctx):
    dp, u, sj, nz = _bruss_case(nls, ctx, 2, 64)
    for bad in (dict(theta=-0.1), dict(theta=1.5), dict(omega=0.0), dict(presweeps=-1), dict(max_levels=0), dict(max_coarse=0), dict(smooth_omega=0.0)):
        with pytest.raises(nls.abi.B200Error) as e:
            nls.SparseAMG.smoothed_aggregation(ctx, dp.n, sj.colptr, sj.rowval, 1, **bad)
        assert e.value.code == nls.abi.ERR_INVALID and "options out of range" in str(e.value), bad
    amg = nls.SparseAMG.smoothed_aggregation(ctx, dp.n, sj.colptr, sj.rowval, 1)
    with pytest.raises(nls.abi.B200Error) as e:           # a refresh needs a hierarchy
        amg.setup(nz, rebuild=False)
    assert e.value.code == nls.abi.ERR_INVALID
    amg = nls.SparseAMG.smoothed_aggregation(ctx, dp.n, sj.colptr, sj.rowval, 1, max_levels=1)
    with pytest.raises(nls.abi.B200Error) as e:           # one level of 8192 unknowns: above the dense cap
        amg.setup(nz)
    assert e.value.code == nls.abi.ERR_UNSUPPORTED and "8192" in str(e.value) and "raise max_levels" in str(e.value)
    rs = nls.SparseAMG(ctx, dp.n, sj.colptr, sj.rowval, 1)   # T exists on smoothed-aggregation handles only
    assert rs.setup(nz) == 0
    L = nls.abi.lib()
    rowptr = np.zeros(dp.n + 1, dtype=np.int32)
    assert L.b200_amg_export(rs._h, 0, nls.abi.AMG_EXPORT_T, rowptr.ctypes.data_as(C.c_void_p), None, None) == nls.abi.ERR_INVALID
    assert "smoothed-aggregation handles only" in L.b200_last_error(ctx.handle).decode()


def test_newton_refuses_sa_where_it_cannot_run(nls, ctx):
    N = 8
    f = nls.Brusselator2D(N)
    dp = nls._DeviceProblem(ctx, nls.NonlinearProblem(f, None, (3.4, 1.0, 10.0), ctx=ctx))
    u0 = dp.u0(nls.abi.U0_PERTURBED_Z).to_host()
    prob = nls.NonlinearProblem(f, u0, (3.4, 1.0, 10.0), ctx=ctx)
    with pytest.raises(nls.abi.B200Error) as e:
        nls.solve(prob, nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(precs=nls.SmoothedAggregationAMG("left"))), abstol=1e-8)
    assert e.value.code == nls.abi.ERR_INVALID and "concrete_jac = true" in str(e.value)
    with pytest.raises(nls.abi.B200Error) as e:
        nls.solve(prob, nls.PseudoTransient(concrete_jac=True, linsolve=nls.KrylovJL_GMRES(precs=nls.SmoothedAggregationAMG("right"))), abstol=1e-8)
    assert e.value.code == nls.abi.ERR_UNSUPPORTED and "PseudoTransient" in str(e.value)
    L = nls.abi.lib()
    for linsolve in (nls.abi.LINSOLVE_DENSE_LU, nls.abi.LINSOLVE_SPARSE_LU):
        o = nls.abi.NewtonOpts()
        L.b200_newton_opts_default(C.byref(o))
        o.linsolve, o.precond = linsolve, nls.abi.PRECOND_SA_AMG_RIGHT
        h = C.c_void_p()
        assert L.b200_newton_create(dp.handle, C.byref(o), C.byref(h)) == nls.abi.ERR_INVALID
    o = nls.abi.NewtonOpts()
    L.b200_newton_opts_default(C.byref(o))
    o.precond = nls.abi.PRECOND_SA_AMG_RIGHT + 1
    assert L.b200_newton_create(dp.handle, C.byref(o), C.byref(C.c_void_p())) == nls.abi.ERR_INVALID
    assert "unknown preconditioner" in L.b200_last_error(ctx.handle).decode()
    u = ctx.to_device(u0)
    for kind in (nls.abi.PRECOND_SA_AMG_LEFT, nls.abi.PRECOND_SA_AMG_RIGHT):
        assert L.b200_linop_precond(dp.handle, u.ptr, kind, C.byref(C.c_void_p())) == nls.abi.ERR_INVALID
        assert "b200_amg_create_sa" in L.b200_last_error(ctx.handle).decode()


def _compare(nls, sol0, sol1):
    assert sol0.retcode == sol1.retcode == nls.ReturnCode.Success
    assert np.abs(sol1.u - sol0.u).max() <= 1e-6 * max(1.0, np.abs(sol0.u).max())
    assert _iters_per_step(sol1) < _iters_per_step(sol0)
    assert sol1.stats.nfactors == sol0.stats.nfactors == 0


@pytest.mark.parametrize("side", ["left", "right"])
def test_newton_raphson_2d_with_sa(nls, ctx, side):
    N = 32
    f = nls.Brusselator2D(N)
    u0 = nls._DeviceProblem(ctx, nls.NonlinearProblem(f, None, (3.4, 1.0, 10.0), ctx=ctx)).u0(nls.abi.U0_PERTURBED_Z).to_host()
    prob = nls.NonlinearProblem(f, u0, (3.4, 1.0, 10.0), ctx=ctx)
    s0 = nls.solve(prob, nls.NewtonRaphson(concrete_jac=True, linsolve=nls.KrylovJL_GMRES()), abstol=1e-8)
    s1 = nls.solve(prob, nls.NewtonRaphson(concrete_jac=True, linsolve=nls.KrylovJL_GMRES(precs=nls.SmoothedAggregationAMG(side), **_krylov_kw(side))),
                   abstol=1e-8)
    _compare(nls, s0, s1)


@pytest.mark.parametrize("side", ["left", "right"])
def test_trust_region_3d_with_sa(nls, ctx, side):
    N = 16
    f = nls.Brusselator3D(N)
    u0 = nls._DeviceProblem(ctx, nls.NonlinearProblem(f, None, (3.4, 1.0, 10.0), ctx=ctx)).u0(nls.abi.U0_PERTURBED_Z).to_host()
    fs = nls.NonlinearFunction(f, sparsity=nls.TracerSparsityDetector())
    prob = nls.NonlinearProblem(fs, u0, (3.4, 1.0, 10.0), ctx=ctx)
    s0 = nls.solve(prob, nls.TrustRegion(linsolve=nls.KrylovJL_GMRES(orth="mgs")), abstol=1e-8)
    s1 = nls.solve(prob, nls.TrustRegion(linsolve=nls.KrylovJL_GMRES(orth="mgs", precs=nls.SmoothedAggregationAMG(side), **_krylov_kw(side))), abstol=1e-8)
    _compare(nls, s0, s1)


@pytest.mark.parametrize("side", ["left", "right"])
def test_user_callback_with_jac_prototype_and_sa(nls, ctx, side):
    fn, u0 = _user_reaction_diffusion(nls, ctx, 32)
    prob = nls.NonlinearProblem(fn, u0, None, ctx=ctx)
    s0 = nls.solve(prob, nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES()), abstol=1e-9)
    s1 = nls.solve(prob, nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(precs=nls.SmoothedAggregationAMG(side), **_krylov_kw(side))), abstol=1e-9)
    _compare(nls, s0, s1)
    assert np.abs(s1.u - 1.0).max() < 1e-8


def test_config4_structure(nls, ctx):
    """3D Brusselator N = 100 (two million unknowns): every coarse pattern is that of P' A P and A_c x = P' (A (P x)) to 1e-12,
    and level 0's aggregates come from a distance-2 maximal independent set of the strength graph."""
    dp, u, sj, nz = _bruss_case(nls, ctx, 3, 100)
    n = dp.n
    amg = nls.SparseAMG.smoothed_aggregation(ctx, n, sj.colptr, sj.rowval, 1)
    assert amg.setup(nz) == 0
    ns, _ = amg.levels()
    assert len(ns) >= 3 and ns[-1] <= 4096
    one = lambda M: sp.csr_matrix((np.ones(M.nnz), M.indices, M.indptr), shape=M.shape)  # noqa: E731
    rng = np.random.default_rng(3)
    lv = amg.level(0)
    A0, T0 = _csr(lv["A"]), lv["T"]
    for l in range(len(ns) - 1):
        nxt = amg.level(l + 1)
        A, P = _csr(lv["A"]), sp.csr_matrix(lv["P"], shape=(ns[l], ns[l + 1]))
        S = (one(P).T @ one(A) @ one(P)).tocsr()
        S.sort_indices()
        assert np.array_equal(S.indptr, nxt["A"][2]) and np.array_equal(S.indices, nxt["A"][1])
        x = rng.standard_normal(ns[l + 1])
        ref = P.T @ (A @ (P @ x))
        assert np.abs(_csr(nxt["A"]) @ x - ref).max() <= 1e-12 * np.abs(ref).max()
        lv = nxt
    # level 0: the restated MIS-2 of the strength graph; roots numbered in index order as T's columns
    G = sa.strength_graph(A0)
    state, _ = sa.mis2(G)
    root = state == sa.IN
    agg = -np.ones(n, dtype=np.int64)
    agg[np.repeat(np.arange(n), np.diff(T0[2]))] = T0[1]
    assert root.sum() == ns[1] and np.array_equal(agg[root], np.arange(ns[1]))
    near = G @ root.astype(np.float64)                               # adjacent roots per node
    assert not near[root].any() and near.max() <= 1                 # no two roots within distance 2
    iso = np.diff(G.indptr) == 0
    covered = root | (near > 0) | ((G @ (near > 0).astype(np.float64)) > 0)
    assert covered[~iso].all()                                       # maximal
    assert (agg[~iso] >= 0).all() and (agg[iso] < 0).all()          # every non-isolated node aggregated
