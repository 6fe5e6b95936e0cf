"""Independent whole-array restatement (NumPy / scipy.sparse) of the classical Ruge-Stueben AMG of csrc/amg.cu, written from the
rules of DESIGN.md §4h, not from the CUDA: strength, the first-pass C/F splitting, direct interpolation, Galerkin coarse
operators, the V(nu1, nu2) cycle with damped Jacobi, and the frozen-splitting refresh.  Test infrastructure only.

Matrices are scipy CSR with sorted indices and every structural entry kept (explicit zeros included): patterns here are
structural, as in the library, so Galerkin patterns come from products of the 0/1 patterns, never from the values."""
import heapq

import numpy as np
import scipy.sparse as sp


def csr_of_csc(n, colptr, rowval, nzval, index_base=1):
    """CSR (sorted indices, explicit zeros kept) of a CSC matrix given as arrays."""
    A = sp.csc_matrix((np.asarray(nzval, dtype=np.float64), np.asarray(rowval, dtype=np.int64) - index_base,
                       np.asarray(colptr, dtype=np.int64) - index_base), shape=(n, n)).tocsr()
    A.sort_indices()
    return A


def _rows(A):
    return np.repeat(np.arange(A.shape[0]), np.diff(A.indptr))


def strength(A, theta=0.25):
    """Boolean mask over A's CSR positions: j strongly influences i (j != i) when |a_ij| >= theta max_{k != i} |a_ik|; a row whose
    off-diagonal entries are all zero has no strong connection; a stored 0.0 is never strong."""
    rows, cols, v = _rows(A), A.indices, A.data
    off = cols != rows
    mx = np.zeros(A.shape[0])
    np.maximum.at(mx, rows[off], np.abs(v[off]))
    return off & (v != 0.0) & (mx[rows] > 0.0) & (np.abs(v) >= theta * mx[rows])


def split(A, strong):
    """The Ruge-Stueben first pass; True at C points.  Isolated points (no strong connection either way) are F; then the
    unassigned point of largest lambda (ties: smallest index) becomes C, the unassigned points it strongly influences become F,
    and every unassigned point that strongly influences a new F point gains one in lambda."""
    n = A.shape[0]
    rows = _rows(A)
    S = sp.csr_matrix((np.ones(int(strong.sum())), (rows[strong], A.indices[strong])), shape=(n, n))   # S[i, j]: j influences i
    ST = S.T.tocsr()
    S.sort_indices(); ST.sort_indices()
    state = np.zeros(n, dtype=np.int8)                 # 0 unassigned, 1 C, 2 F
    state[(np.diff(S.indptr) == 0) & (np.diff(ST.indptr) == 0)] = 2
    lam = np.diff(ST.indptr).astype(np.int64)
    heap = [(-int(lam[i]), i) for i in range(n) if state[i] == 0]
    heapq.heapify(heap)
    while heap:
        l, i = heapq.heappop(heap)
        if state[i] != 0 or -l != lam[i]:
            continue
        state[i] = 1
        for j in ST.indices[ST.indptr[i]:ST.indptr[i + 1]]:
            if state[j] != 0:
                continue
            state[j] = 2
            for k in S.indices[S.indptr[j]:S.indptr[j + 1]]:
                if state[k] == 0:
                    lam[k] += 1
                    heapq.heappush(heap, (-int(lam[k]), int(k)))
    return state == 1


def interpolation(A, ci):
    """Direct interpolation; `ci` marks the positions of A that are strong C-neighbours (the F rows' interpolatory set).  C rows
    of P are unit rows; for F rows alpha (negative) and beta (positive) scale the strong C entries, with the positive
    off-diagonal sum lumped into a_ii when C_i holds no positive entry."""
    n = A.shape[0]
    rows, cols, v = _rows(A), A.indices, A.data
    off = cols != rows
    d = np.zeros(n)
    np.add.at(d, rows[~off], v[~off])
    an, ap, sn, spos = (np.zeros(n) for _ in range(4))
    np.add.at(an, rows[off & (v < 0)], v[off & (v < 0)])
    np.add.at(ap, rows[off & (v > 0)], v[off & (v > 0)])
    np.add.at(sn, rows[ci & (v < 0)], v[ci & (v < 0)])
    np.add.at(spos, rows[ci & (v > 0)], v[ci & (v > 0)])
    alpha = np.divide(an, sn, out=np.zeros(n), where=sn != 0)
    beta = np.divide(ap, spos, out=np.zeros(n), where=spos != 0)
    d = np.where(spos == 0, d + ap, d)
    return rows[ci], cols[ci], -np.where(v[ci] < 0, alpha[rows[ci]], beta[rows[ci]]) * v[ci] / d[rows[ci]]


def build_p(A, cf, ci):
    n = A.shape[0]
    cidx = np.cumsum(cf) - 1
    r, c, w = interpolation(A, ci)
    C = np.nonzero(cf)[0]
    P = sp.csr_matrix((np.concatenate([np.ones(len(C)), w]), (np.concatenate([C, r]), cidx[np.concatenate([C, c])])), shape=(n, int(cf.sum())))
    P.sort_indices()
    return P


def galerkin(A, P):
    """R A P with R = P' on the structural pattern of the product (values by scipy, read at the pattern's positions)."""
    one = lambda M: sp.csr_matrix((np.ones(M.nnz), M.indices, M.indptr), shape=M.shape)  # noqa: E731
    S = (one(P).T @ one(A) @ one(P)).tocsr()
    S.sort_indices()
    V = (P.T @ (A @ P)).tocsr()
    rows = _rows(S)
    vals = np.asarray(V[rows, S.indices]).ravel() if S.nnz else np.zeros(0)
    Ac = sp.csr_matrix((vals, S.indices.copy(), S.indptr.copy()), shape=S.shape)
    return Ac


class Hierarchy:
    """levels[l] = dict(A, P, cf, ci) for every level but the coarsest; coarse = the coarsest A; coarse_inv its inverse."""

    def __init__(self, A, theta=0.25, omega=2.0 / 3.0, presweeps=1, postsweeps=1, max_levels=10, max_coarse=10, frozen=None):
        self.omega, self.pre, self.post = omega, presweeps, postsweeps
        self.levels = []
        A = A.tocsr()
        while True:
            l = len(self.levels)
            if frozen is not None:
                if l == len(frozen.levels):
                    break
                cf, ci = frozen.levels[l]["cf"], frozen.levels[l]["ci"]
            else:
                if A.shape[0] <= max_coarse or l + 1 >= max_levels:
                    break
                strong = strength(A, theta)
                cf = split(A, strong)
                if cf.sum() == 0 or cf.sum() == A.shape[0]:
                    break
                ci = strong & cf[A.indices] & ~cf[_rows(A)]   # strong C-neighbours of F points
            P = build_p(A, cf, ci)
            self.levels.append(dict(A=A, P=P, cf=cf, ci=ci))
            A = galerkin(A, P)
        self.coarse = A
        self._coarse_inv = None

    @property
    def coarse_inv(self):
        """The coarsest level's explicit inverse (formed on first use: a singular coarsest level only fails the cycle)."""
        if self._coarse_inv is None:
            self._coarse_inv = np.linalg.inv(self.coarse.toarray())
        return self._coarse_inv

    def refresh(self, A0):
        """The same splitting and patterns, every value recomputed from the new level-0 values (what a device refresh does)."""
        return Hierarchy(A0, omega=self.omega, presweeps=self.pre, postsweeps=self.post, frozen=self)

    def sizes(self):
        return [L["A"].shape[0] for L in self.levels] + [self.coarse.shape[0]]

    def nnz(self):
        return [L["A"].nnz for L in self.levels] + [self.coarse.nnz]

    def operator_complexity(self):
        z = self.nnz()
        return sum(z) / z[0]

    def cycle(self, b, l=0):
        """One V(pre, post) cycle from x = 0 on level l."""
        if l == len(self.levels):
            return self.coarse_inv @ b
        A, P = self.levels[l]["A"], self.levels[l]["P"]
        dinv = 1.0 / A.diagonal()
        x = np.zeros_like(b)
        for _ in range(self.pre):
            x = x + self.omega * dinv * (b - A @ x)
        x = x + P @ self.cycle(P.T @ (b - A @ x), l + 1)
        for _ in range(self.post):
            x = x + self.omega * dinv * (b - A @ x)
        return x
