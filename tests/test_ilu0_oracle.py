"""The NumPy restatement of ILU(0) (oracle/ilu0_numpy.py) against the properties that define it: L U reproduces A on the
pattern, it is the exact LU on patterns closed under fill, and its level counts on the Brusselator patterns are the
structural 2N (2D) and 3N - 1 (3D)."""
import numpy as np
import pytest

from oracle import ilu0_numpy as il

EPS = np.finfo(np.float64).eps


def _csc(A, index_base=1):
    """CSC of the structure of the dense matrix A (explicit entries where A != 0, plus the diagonal)."""
    n = A.shape[0]
    S = (A != 0) | np.eye(n, dtype=bool)
    colptr, rowval, nzval = [0], [], []
    for c in range(n):
        r = np.nonzero(S[:, c])[0]
        rowval.extend(r.tolist())
        nzval.extend(A[r, c].tolist())
        colptr.append(len(rowval))
    return np.array(colptr) + index_base, np.array(rowval) + index_base, np.array(nzval)


def _dd_matrix(rng, n, mask):
    A = np.where(mask, rng.uniform(-1.0, 1.0, (n, n)), 0.0)
    np.fill_diagonal(A, 0.0)
    np.fill_diagonal(A, np.abs(A).sum(axis=1) + 1.0 + rng.uniform(0, 1, n))
    return A


def _dense_lu_nopivot(A):
    n = A.shape[0]
    W = A.copy()
    for k in range(n):
        W[k + 1:, k] /= W[k, k]
        W[k + 1:, k + 1:] -= np.outer(W[k + 1:, k], W[k, k + 1:])
    return np.tril(W, -1) + np.eye(n), np.triu(W)


@pytest.mark.parametrize("n,density,base", [(40, 0.08, 1), (120, 0.03, 0), (200, 0.02, 1)])
def test_lu_reproduces_a_on_the_pattern(n, density, base):
    rng = np.random.default_rng(n)
    A = _dd_matrix(rng, n, rng.uniform(size=(n, n)) < density)
    colptr, rowval, nz = _csc(A, base)
    f, info = il.ilu0(n, colptr, rowval, nz, base)
    assert info == 0
    L, U = il.dense_factors(n, colptr, rowval, f, base)
    S = (A != 0) | np.eye(n, dtype=bool)
    err = np.abs(L @ U - A)[S]
    bound = 2.0 * n * EPS * (np.abs(L) @ np.abs(U))[S] + 1e-300
    assert (err <= bound).all()
    # the restatement's solve is the two triangular solves with its own factors
    b = rng.standard_normal(n)
    x = il.solve(n, colptr, rowval, f, b, base)
    assert np.allclose(x, np.linalg.solve(U, np.linalg.solve(L, b)), rtol=1e-12, atol=1e-12 * np.abs(x).max())


@pytest.mark.parametrize("kind,n,w", [("tridiagonal", 300, 1), ("band", 120, 5), ("band", 64, 63)])
def test_closed_patterns_give_the_exact_lu(kind, n, w):
    rng = np.random.default_rng(7 + w)
    i, j = np.indices((n, n))
    A = _dd_matrix(rng, n, np.abs(i - j) <= w)
    colptr, rowval, nz = _csc(A)
    f, info = il.ilu0(n, colptr, rowval, nz)
    assert info == 0
    L, U = il.dense_factors(n, colptr, rowval, f)
    L0, U0 = _dense_lu_nopivot(A)
    assert np.abs(L - L0).max() <= 1e-14 * np.abs(L0).max()
    assert np.abs(U - U0).max() <= 1e-14 * np.abs(U0).max()


@pytest.mark.parametrize("dim,N,expect", [(2, 32, 64), (2, 64, 128), (3, 16, 47), (3, 24, 71), (2, 5, 10), (3, 7, 20)])
def test_brusselator_level_counts(po, dim, N, expect):
    P = po.OracleProblem.bruss2d(N) if dim == 2 else po.OracleProblem.bruss3d(N)
    colptr, rowval = P.pattern(1)
    assert expect == (2 * N if dim == 2 else 3 * N - 1)
    assert il.level_counts(P.n, colptr, rowval, 1) == (expect, expect)


def test_zero_pivot_and_missing_diagonal():
    A = np.array([[1.0, 1.0, 0.0], [1.0, 1.0, 0.0], [0.0, 0.0, 0.0]])
    colptr, rowval, nz = _csc(A)
    _, info = il.ilu0(3, colptr, rowval, nz)
    assert info == 2                      # u_22 = 1 - 1 * 1 = 0; row 3 is also zero, the first one is reported
    with pytest.raises(ValueError, match="row 1"):
        il.ilu0(2, np.array([1, 2, 3]), np.array([1, 1]), np.ones(2))
