"""The NumPy restatement of the smoothed-aggregation AMG (oracle/sa_numpy.py), pinned on the CPU: the distance-2 maximal
independent set, the aggregates, the tentative and smoothed prolongators, Galerkin products, linearity of the cycle, and the
hierarchy sizes and GMRES iteration counts it gives."""
import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components

from oracle import sa_numpy as sa
from test_amg_oracle import bruss, gmres, graph_laplacian, poisson, random_matrix


def _one(M):
    return sp.csr_matrix((np.ones(M.nnz), M.indices, M.indptr), shape=M.shape)


CASES = [lambda: bruss(32), lambda: poisson(64), lambda: random_matrix(800, 3), lambda: graph_laplacian(800, 1) + 0.1 * sp.identity(800)]


@pytest.mark.parametrize("make", CASES)
def test_mis2_and_aggregates(make):
    A = sp.csr_matrix(make())
    G = sa.strength_graph(A)
    assert (G != G.T).nnz == 0 and G.diagonal().sum() == 0
    agg, na, state, _ = sa.aggregate(G)
    root = state == sa.IN
    iso = np.diff(G.indptr) == 0
    G2 = _one(G + G @ G).tolil()
    G2.setdiag(0)
    G2 = G2.tocsr()
    assert G2[root][:, root].nnz == 0                                     # no two roots within distance 2
    reach = np.asarray(G2[:, root].sum(axis=1)).ravel() > 0
    assert (root | reach | iso).all()                                     # maximal
    assert (agg[~iso] >= 0).all() and (agg[iso] < 0).all()                # every non-isolated node aggregated
    assert np.array_equal(agg[root], np.arange(na))                       # roots numbered in index order
    for a in range(na):
        m = np.flatnonzero(agg == a)
        assert connected_components(G[m][:, m], directed=False)[0] == 1   # connected


@pytest.mark.parametrize("make", CASES)
def test_prolongators(make):
    A = sp.csr_matrix(make())
    H = sa.Hierarchy(A)
    b = np.ones(A.shape[0])
    for L in H.levels:
        A, T, P = L["A"], L["T"], L["P"]
        TT = (T.T @ T).toarray()
        assert np.allclose(TT, np.eye(T.shape[1]), rtol=0, atol=1e-14)   # orthonormal columns
        T_, bc = sa.tentative(L["agg"], T.shape[1], b)
        assert np.allclose(T @ bc, np.where(L["agg"] >= 0, b, 0.0), rtol=1e-14, atol=0)   # T b_c = b on aggregated rows
        Ad, Td = A.toarray(), T.toarray()
        rho = (np.abs(Ad).sum(axis=1) / np.abs(np.diag(Ad))).max()
        Pd = Td - (4.0 / 3.0 / rho) * (Ad @ Td) / np.diag(Ad)[:, None]
        assert np.abs(P.toarray() - Pd).max() <= 1e-13 * max(1.0, np.abs(Pd).max())
        S = (_one(A) @ _one(T)).tocsr()
        S.sort_indices()
        assert np.array_equal(P.indptr, S.indptr) and np.array_equal(P.indices, S.indices)
        b = bc
    Ls = H.levels + [None]
    for l, L in enumerate(H.levels):
        Ac = Ls[l + 1]["A"] if Ls[l + 1] is not None else H.coarse
        Pd = L["P"].toarray()
        ref = Pd.T @ L["A"].toarray() @ Pd
        assert np.abs(Ac.toarray() - ref).max() <= 1e-12 * np.abs(ref).max()


def test_cycle_is_linear():
    A = bruss(32)
    H = sa.Hierarchy(A)
    rng = np.random.default_rng(0)
    x, y = rng.standard_normal((2, A.shape[0]))
    lhs = H.cycle(2.0 * x - 3.0 * y)
    assert np.abs(lhs - (2.0 * H.cycle(x) - 3.0 * H.cycle(y))).max() <= 1e-11 * np.abs(lhs).max()


def test_frozen_refresh_at_the_same_values_is_the_rebuild():
    A = bruss(32)
    H = sa.Hierarchy(A)
    R = H.refresh(A)
    assert R.sizes() == H.sizes()
    for L, M in zip(H.levels, R.levels):
        assert (L["P"] != M["P"]).nnz == 0 and (L["A"] != M["A"]).nnz == 0


@pytest.mark.parametrize("name,make,sizes,its", [
    ("bruss32", lambda: bruss(32), [2048, 286, 29, 3], (17, 23)),
    ("poisson64", lambda: poisson(64), [4096, 592, 71, 11, 2], (21, 22)),
    ("laplacian", lambda: graph_laplacian(2000, 4) + 0.1 * sp.identity(2000), [2000, 216, 3], (16, 16)),   # one isolated row
])
def test_hierarchy_sizes_and_iterations(name, make, sizes, its):
    A = sp.csr_matrix(make())
    H = sa.Hierarchy(A)
    b = np.random.default_rng(0).standard_normal(A.shape[0])
    left, right = gmres(A, b, H.cycle, "left")[0], gmres(A, b, H.cycle, "right")[0]
    assert H.sizes() == sizes and (left, right) == its
    assert (H.levels[0]["agg"] < 0).any() == (name == "laplacian")
