"""The library's host splitting (b200_amg_split) against the NumPy restatement, element for element (no device needed)."""
import numpy as np
import pytest
import scipy.sparse as sp

from oracle import amg_numpy as am


def _csc(A, base):
    A = sp.csc_matrix(A)
    A.sort_indices()
    return A.indptr.astype(np.int64) + base, A.indices.astype(np.int64) + base, A.data.astype(np.float64)


def _check(nls, n, colptr, rowval, nzval, base, theta=0.25):
    cf_lib, nc = nls.amg_split(n, colptr, rowval, nzval, base, theta)
    A = am.csr_of_csc(n, colptr, rowval, nzval, base)
    cf = am.split(A, am.strength(A, theta))
    assert np.array_equal(cf_lib, cf) and nc == int(cf.sum())
    return cf


@pytest.mark.parametrize("N", [8, 32])
def test_brusselator_2d(nls, golden, N):
    n = 2 * N * N
    cf = _check(nls, n, golden["colptr_%d" % N], golden["rowval_%d" % N], golden["nzval_%d" % N], 1)
    assert cf.sum() == n // 2


def test_brusselator_3d(nls, po):
    P3 = po.OracleProblem.bruss3d(10)
    colptr, rowval = P3.pattern(1)
    colors, ncolors = po.coloring_column(P3.n, colptr, rowval, 1)
    nz = P3.sparse_jac(P3.u0(1), colptr, rowval, colors, ncolors, 1)   # the Jacobian at the perturbed initial condition
    _check(nls, P3.n, colptr, rowval, nz, 1)


@pytest.mark.parametrize("seed", range(8))
@pytest.mark.parametrize("base", [0, 1])
def test_random_both_signs(nls, seed, base):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(5, 400))
    A = sp.random(n, n, density=min(1.0, 6.0 / n), random_state=rng, data_rvs=lambda k: rng.standard_normal(k)).tolil()
    iso = rng.random(n) < 0.1
    A[np.nonzero(iso)[0], :] = 0.0
    A[:, np.nonzero(iso)[0]] = 0.0
    A.setdiag(rng.standard_normal(n))
    A = A.tocsc()
    colptr, rowval, nz = _csc(A, base)
    nz[rng.random(len(nz)) < 0.05] = 0.0          # stored zeros are never strong
    _check(nls, n, colptr, rowval, nz, base, theta=[0.25, 0.5, 0.1][seed % 3])


@pytest.mark.parametrize("base", [0, 1])
def test_empty_and_isolated_rows(nls, base):
    n = 6
    # column 0: rows 0, 1; column 1: rows 0, 1; column 2: nothing; column 3: row 3 only; columns 4, 5: a coupled pair
    colptr = np.array([0, 2, 4, 4, 5, 7, 9], dtype=np.int64) + base
    rowval = np.array([0, 1, 0, 1, 3, 4, 5, 4, 5], dtype=np.int64) + base
    nz = np.array([2.0, -1.0, -1.0, 2.0, 1.0, 3.0, -1.0, -1.0, 3.0])
    cf = _check(nls, n, colptr, rowval, nz, base)
    assert not cf[2] and not cf[3]                 # empty row and column; a row with only its diagonal
    assert cf[0] != cf[1] and cf[4] != cf[5]
