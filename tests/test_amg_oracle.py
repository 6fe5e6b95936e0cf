"""The NumPy restatement of the Ruge-Stueben AMG (oracle/amg_numpy.py), pinned on the CPU: structure of P, the splitting against
a naive statement of the rule, Galerkin products, linearity of the cycle, and the h-independence the preconditioner is for."""
import os

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import amg_numpy as am

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def gmres(A, b, M=None, side="right", tol=1e-10, maxit=400):
    """Unrestarted GMRES (MGS Arnoldi) from x = 0; returns (iterations, x).  Right preconditioning: the residual it monitors is
    the true one; left: the preconditioned one."""
    M = M or (lambda v: v)
    op = (lambda v: A @ M(v)) if side == "right" else (lambda v: M(A @ v))
    r0 = b if side == "right" else M(b)
    beta = np.linalg.norm(r0)
    V = [r0 / beta]
    H = np.zeros((maxit + 1, maxit))
    for k in range(maxit):
        w = op(V[k])
        for j in range(k + 1):
            H[j, k] = V[j] @ w
            w = w - H[j, k] * V[j]
        H[k + 1, k] = np.linalg.norm(w)
        e1 = np.zeros(k + 2)
        e1[0] = beta
        y = np.linalg.lstsq(H[:k + 2, :k + 1], e1, rcond=None)[0]
        if np.linalg.norm(e1 - H[:k + 2, :k + 1] @ y) <= tol * beta or H[k + 1, k] == 0.0:
            z = np.array(V).T @ y
            return k + 1, (M(z) if side == "right" else z)
        V.append(w / H[k + 1, k])
    raise AssertionError("GMRES did not converge in %d iterations" % maxit)


def poisson(N, periodic=False):
    T = sp.diags([-1.0, 2.0, -1.0], [-1, 0, 1], shape=(N, N), format="lil")
    if periodic:
        T[0, N - 1] = T[N - 1, 0] = -1.0
    I = sp.identity(N)
    A = (sp.kron(I, T) + sp.kron(T, I)).tocsr()
    A.sort_indices()
    return A


def graph_laplacian(n, seed):
    rng = np.random.default_rng(seed)
    W = sp.random(n, n, density=4.0 / n, random_state=rng, data_rvs=lambda k: rng.uniform(0.1, 2.0, k))
    W = ((W + W.T) * 0.5).tolil()
    W.setdiag(0.0)
    W = W.tocsr()
    W.eliminate_zeros()
    L = (sp.diags(np.asarray(W.sum(axis=1)).ravel()) - W).tocsr()
    L = (L + sp.diags(np.zeros(n))).tocsr()  # keep the diagonal structural, also on isolated rows
    L.sort_indices()
    return L


def random_matrix(n, seed, isolated=0.1):
    """Non-symmetric, both signs, some rows and columns holding nothing but the diagonal."""
    rng = np.random.default_rng(seed)
    A = sp.random(n, n, density=min(1.0, 5.0 / n), random_state=rng, data_rvs=lambda k: rng.standard_normal(k)).tolil()
    iso = rng.random(n) < isolated
    A[np.nonzero(iso)[0], :] = 0.0
    A[:, np.nonzero(iso)[0]] = 0.0
    A.setdiag(4.0 + rng.random(n))
    A = A.tocsr()
    A.sort_indices()
    return A


def bruss(N):
    d = np.load(os.path.join(ROOT, "tests", "golden", "brusselator_golden.npz"))
    return am.csr_of_csc(2 * N * N, d["colptr_%d" % N], d["rowval_%d" % N], d["nzval_%d" % N])


def naive_split(A, theta=0.25):
    """Rule 2 word for word on dense arrays, O(n^2) per pick."""
    n = A.shape[0]
    D = A.toarray()
    S = np.zeros((n, n), dtype=bool)          # S[i, j]: j strongly influences i
    for i in range(n):
        off = [abs(D[i, k]) for k in range(n) if k != i]
        mx = max(off) if off else 0.0
        if mx > 0.0:
            for j in range(n):
                S[i, j] = j != i and D[i, j] != 0.0 and abs(D[i, j]) >= theta * mx
    state = ["U"] * n
    for i in range(n):
        if not S[i, :].any() and not S[:, i].any():
            state[i] = "F"
    lam = [int(S[:, i].sum()) for i in range(n)]
    while "U" in state:
        best = max((i for i in range(n) if state[i] == "U"), key=lambda i: (lam[i], -i))
        state[best] = "C"
        for j in range(n):
            if S[j, best] and state[j] == "U":
                state[j] = "F"
                for k in range(n):
                    if S[j, k] and state[k] == "U":
                        lam[k] += 1
    return np.array([s == "C" for s in state])


@pytest.mark.parametrize("seed", range(6))
def test_split_equals_the_naive_rule(seed):
    n = [7, 30, 64, 150, 220, 300][seed]
    A = random_matrix(n, seed)
    assert np.array_equal(am.split(A, am.strength(A)), naive_split(A))


def _levels_of(A, **kw):
    H = am.Hierarchy(A, **kw)
    assert len(H.levels) >= 1
    return H


@pytest.mark.parametrize("make", [lambda: poisson(24), lambda: bruss(8), lambda: random_matrix(200, 3)])
def test_p_structure(make):
    A = make()
    for L in _levels_of(A).levels:
        A, P, cf = L["A"], L["P"], L["cf"]
        strong = am.strength(A)
        rows = np.repeat(np.arange(A.shape[0]), np.diff(A.indptr))
        C = np.nonzero(cf)[0]
        # C rows are unit rows at their coarse index
        assert np.array_equal(np.diff(P.indptr)[C], np.ones(len(C)))
        assert np.array_equal(P.indices[P.indptr[C]], np.arange(len(C))) and np.all(P.data[P.indptr[C]] == 1.0)
        # exactly the isolated points have empty rows; every F point with a strong dependence has a strong C-neighbour
        dep = np.bincount(rows[strong], minlength=A.shape[0]) > 0
        infl = np.bincount(A.indices[strong], minlength=A.shape[0]) > 0
        assert np.array_equal(np.diff(P.indptr) == 0, ~dep & ~infl)
        has_c = np.bincount(rows[strong & cf[A.indices]], minlength=A.shape[0]) > 0
        assert np.all(has_c[~cf & dep])


@pytest.mark.parametrize("A", [poisson(16, periodic=True), poisson(33, periodic=True), graph_laplacian(300, 1), graph_laplacian(500, 2)],
                         ids=["periodic16", "periodic33", "graph300", "graph500"])
def test_rows_of_p_sum_to_one_on_zero_row_sum_m_matrices(A):
    H = am.Hierarchy(A, max_coarse=4)
    L = H.levels[0]
    P, cf, A0 = L["P"], L["cf"], L["A"]
    s = np.asarray(P.sum(axis=1)).ravel()
    nonempty = np.diff(P.indptr) > 0
    assert np.abs(s[nonempty] - 1.0).max() <= 1e-12


@pytest.mark.parametrize("make", [lambda: bruss(8), lambda: poisson(20), lambda: random_matrix(250, 5)])
def test_galerkin_equals_dense_product(make):
    H = _levels_of(make())
    for l, L in enumerate(H.levels):
        Ac = H.levels[l + 1]["A"] if l + 1 < len(H.levels) else H.coarse
        P = L["P"].toarray()
        ref = P.T @ L["A"].toarray() @ P
        assert np.abs(Ac.toarray() - ref).max() <= 1e-13 * max(1.0, np.abs(ref).max())


def test_cycle_is_linear():
    A = bruss(32)
    H = am.Hierarchy(A)
    rng = np.random.default_rng(0)
    x, y = rng.standard_normal(A.shape[0]), rng.standard_normal(A.shape[0])
    lhs = H.cycle(2.0 * x - 3.0 * y)
    rhs = 2.0 * H.cycle(x) - 3.0 * H.cycle(y)
    assert np.abs(lhs - rhs).max() <= 1e-12 * np.abs(rhs).max()


def test_frozen_refresh_at_the_same_values_is_the_rebuild():
    A = bruss(32)
    H = am.Hierarchy(A)
    R = H.refresh(A)
    assert R.sizes() == H.sizes()
    for L, M in zip(H.levels, R.levels):
        assert np.array_equal(L["P"].indices, M["P"].indices) and np.array_equal(L["P"].data, M["P"].data)
    assert np.array_equal(H.coarse.data, R.coarse.data)


def test_brusselator_hierarchy():
    H = am.Hierarchy(bruss(32))
    assert H.sizes() == [2048, 1024, 256, 64, 16, 4]
    assert abs(H.operator_complexity() - 2.988) < 1e-3


def test_poisson_iterations_are_h_independent():
    its = {}
    for N in (32, 64, 128):
        A = poisson(N)
        H = am.Hierarchy(A)
        b = np.random.default_rng(N).standard_normal(A.shape[0])
        its[N], x = gmres(A, b, M=H.cycle)
        assert np.linalg.norm(b - A @ x) <= 1e-9 * np.linalg.norm(b)
    assert its[128] <= 1.5 * its[32], its


# GMRES iterations to a relative residual of 1e-10 on the 2D N = 32 Brusselator Jacobian at u0 (DESIGN.md §4h keeps them):
# unpreconditioned, and one V(1,1) cycle on either side for three Jacobi dampings
BRUSS32_ITERS = {"none": 181, ("left", 0.5): 9, ("left", 2.0 / 3.0): 8, ("left", 0.8): 8,
                 ("right", 0.5): 12, ("right", 2.0 / 3.0): 10, ("right", 0.8): 11}


def test_brusselator_iteration_counts_by_omega():
    A = bruss(32)
    b = np.random.default_rng(0).standard_normal(A.shape[0])
    got = {"none": gmres(A, b)[0]}
    for om in (0.5, 2.0 / 3.0, 0.8):
        H = am.Hierarchy(A, omega=om)
        for side in ("left", "right"):
            got[(side, om)] = gmres(A, b, M=H.cycle, side=side)[0]
    assert got == BRUSS32_ITERS
