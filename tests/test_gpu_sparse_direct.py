"""The sparse direct route (csrc/sparse_lu.cu: reverse Cuthill-McKee ordering, `slu_gbtf2_kernel`, `slu_gbtrs_kernel`) on
matrices that pivot, in every band regime, and the sparse Jacobian plumbing that feeds it (csrc/sparse.cu) on general
user patterns.

References, all on the host:
  * `rcm_perm` restates the ordering of `b200_sparse_lu_create` (symmetrised pattern without its diagonal; per component
    a George-Liu pseudo-peripheral root with at most 8 refinements, ties by minimum degree then lower index; BFS visiting
    neighbours by (degree, index); the whole order reversed).  `lu.bandwidth()` must equal the (kl, ku) it gives.
  * `BandRef` factors the same band array with LAPACK dgbtrf / dgbtrs and forms |L| and |U| of P A = L U.  A device
    solve x must satisfy Higham's Theorem 9.4 restricted to the band, componentwise, with w = 3 (2 kl + ku + 1):
        |b - A x| <= 2 gamma_w P^T |L| |U| |x|                                  (backward)
        |x - x_lapack| <= 2 |A^-1| P^T (gamma_w |L| |U| max(|x|, |x_lapack|))   (forward)
    The residual is summed in long double and |A^-1| comes from the row-equilibrated matrix, so neither check spends
    its margin on its own rounding.
Matrix families (each under one random symmetric permutation, so RCM has real work to do):
  F1 random N(0, 1) bands, F2 bands with no structural diagonal, F3 disconnected dense blocks with isolated vertices,
  F4 lower bands with kl > 1024 whose chosen columns pivot at offsets > 1024 or hold exact ties on different threads,
  F5 kl = ku = 0 and n = 1, F6 the 2D Brusselator at N = 64 (n = 8192).
A test without the GPU marker checks the references against SuperLU and that the pivoting families do pivot, so the
device tests cannot quietly turn into no-pivot tests.

Exact (bit-level) assertions are used only where every correct implementation must agree: repeated solves, in-place
and out-of-place solves, a re-factored handle against a fresh one, index base 0 against base 1, `info` of an exactly
zero column, colourings against the C oracle, and a coloured Jacobian fill (each compressed entry is one product, every
other term an exact zero).
"""
import math
from collections import deque

import numpy as np
import pytest
import scipy.linalg.lapack as lapack
import scipy.sparse as sp

U = 2.0 ** -53
SLU_THREADS = 1024     # threads of the single-CTA band kernels
WIDE_KL = 1040         # F4: lower half-bandwidth, > SLU_THREADS
WIDE_N = 2200         # long enough for RCM to lay the band out end to end
BIG_ROW = 2.0 ** 30    # F4: scale of the row that ties with the first maximum


def gamma(k):
    return k * U / (1.0 - k * U)


# ------------------------------------------------------------------------------------------------ reverse Cuthill-McKee
def sym_adjacency(n, colptr, rowval, base):
    """CSR (indptr, indices) of the symmetrised pattern without its diagonal; indices sorted and unique."""
    cp = np.asarray(colptr, dtype=np.int64) - base
    rv = np.asarray(rowval, dtype=np.int64) - base
    cols = np.repeat(np.arange(n), np.diff(cp))
    off = rv != cols
    r, c = rv[off], cols[off]
    G = sp.csr_matrix((np.ones(2 * r.size), (np.r_[r, c], np.r_[c, r])), shape=(n, n))
    G.sum_duplicates()
    return G.indptr, G.indices


def _last_level(indptr, indices, root):
    """(eccentricity of root, vertices of its last BFS level)."""
    seen = np.zeros(len(indptr) - 1, dtype=bool)
    seen[root] = True
    front, ecc = np.array([root]), 0
    while True:
        nb = np.concatenate([indices[indptr[v]:indptr[v + 1]] for v in front])
        nb = np.unique(nb[~seen[nb]])
        if nb.size == 0:
            return ecc, front
        seen[nb] = True
        front, ecc = nb, ecc + 1


def rcm_perm(n, colptr, rowval, base):
    """The ordering of b200_sparse_lu_create: perm[new] = old."""
    indptr, indices = sym_adjacency(n, colptr, rowval, base)
    deg = np.diff(indptr)
    seen = np.zeros(n, dtype=bool)
    order = []
    for start in range(n):
        if seen[start]:
            continue
        root = start
        ecc, last = _last_level(indptr, indices, root)
        for _ in range(8):
            cand = int(last[np.lexsort((last, deg[last]))[0]])
            e2, last2 = _last_level(indptr, indices, cand)
            if e2 <= ecc:
                break
            root, ecc, last = cand, e2, last2
        seen[root] = True
        q = deque([root])
        while q:
            v = q.popleft()
            order.append(v)
            nb = indices[indptr[v]:indptr[v + 1]]
            nb = nb[~seen[nb]]
            seen[nb] = True
            q.extend(nb[np.lexsort((nb, deg[nb]))].tolist())
    return np.array(order[::-1], dtype=np.int64)


# ------------------------------------------------------------------------------------------------ matrices
class Case:
    """An n x n CSC matrix (0-based colptr / rowval, sorted rows, no duplicates) and its RCM band."""

    def __init__(self, name, n, rows, cols, vals):
        o = np.lexsort((rows, cols))
        self.name, self.n = name, n
        self.rowval, self.cols, self.vals = rows[o].astype(np.int64), cols[o].astype(np.int64), vals[o].astype(np.float64)
        self.colptr = np.r_[0, np.cumsum(np.bincount(self.cols, minlength=n))].astype(np.int64)
        self.perm = rcm_perm(n, self.colptr, self.rowval, 0)
        self.iperm = np.empty(n, dtype=np.int64)
        self.iperm[self.perm] = np.arange(n)
        d = self.iperm[self.rowval] - self.iperm[self.cols]
        self.kl, self.ku = int(max(0, d.max())), int(max(0, -d.min()))

    def csr(self, vals=None):
        return sp.csr_matrix((self.vals if vals is None else vals, (self.rowval, self.cols)), shape=(self.n, self.n))

    def band_array(self, vals=None):
        """LAPACK dgbtrf storage of the RCM-permuted matrix: ab[kl + ku + i - j, j], ldab = 2 kl + ku + 1."""
        ab = np.zeros((2 * self.kl + self.ku + 1, self.n), order="F")
        i, j = self.iperm[self.rowval], self.iperm[self.cols]
        ab[self.kl + self.ku + i - j, j] = self.vals if vals is None else vals
        return ab

    def zeroed(self, column=None, row=None):
        v = self.vals.copy()
        v[(self.cols == column) if column is not None else (self.rowval == row)] = 0.0
        return v

    def __repr__(self):
        return "%s(n=%d, kl=%d, ku=%d)" % (self.name, self.n, self.kl, self.ku)


def _entries(n, offsets):
    """(rows, cols) of the given diagonals i - j = d."""
    rows, cols = [], []
    for d in offsets:
        j = np.arange(max(0, -d), min(n, n - d))
        rows.append(j + d)
        cols.append(j)
    return np.concatenate(rows), np.concatenate(cols)


def _scrambled(name, n, rows, cols, vals, rng):
    """Case of Q A Q^T for a random permutation Q, with duplicate entries of (rows, cols) dropped."""
    key, first = np.unique(rows * n + cols, return_index=True)
    rows, cols, vals = rows[first], cols[first], vals[first]
    q = rng.permutation(n)
    qi = np.empty(n, dtype=np.int64)
    qi[q] = np.arange(n)
    return Case(name, n, qi[rows], qi[cols], vals)


def f1_band(kl, ku, n):
    rng = np.random.default_rng(1000 * kl + 10 * ku + n)
    rows, cols = _entries(n, range(-ku, kl + 1))
    return _scrambled("F1", n, rows, cols, rng.standard_normal(rows.size), rng)


def f2_no_diagonal(n, k=2, shift=5):
    rng = np.random.default_rng(20000 + n)
    rows, cols = _entries(n, [d for d in range(-k, k + 1) if d != 0])
    i = np.arange(n)
    rows, cols = np.r_[rows, i], np.r_[cols, (i + shift) % n]
    return _scrambled("F2", n, rows, cols, rng.standard_normal(rows.size), rng)


def f3_disconnected(n):
    rng = np.random.default_rng(30000 + n)
    rows, cols, start, k = [], [], 0, 0
    while start < n:
        m = min(n - start, 1 if k % 4 == 0 else int(rng.integers(1, 51)))   # every fourth block is an isolated vertex
        r, c = np.meshgrid(np.arange(m), np.arange(m), indexing="ij")
        rows.append(start + r.ravel())
        cols.append(start + c.ravel())
        start, k = start + m, k + 1
    rows, cols = np.concatenate(rows), np.concatenate(cols)
    return _scrambled("F3", n, rows, cols, rng.standard_normal(rows.size), rng)


def f5_diagonal(n):
    rng = np.random.default_rng(50000 + n)
    i = np.arange(n)
    return _scrambled("F5", n, i, i, rng.standard_normal(n) + np.where(rng.random(n) < 0.5, -2.0, 2.0), rng)


# Chosen columns of the wide family, in band coordinates (c = WIDE_C).  "far": the column's maximum sits at offset 1040
# (the second item of thread 16) and everything else in it is ~2^-30, so a pivot search that misses it produces growth
# of ~2^34.  "tie_warp" / "tie_cross": +T and -T at offsets (3, 1026) (threads 3 and 2 of warp 0) or (40, 1030) (thread
# 40 of warp 1, thread 6 of warp 0), with column c zero above its diagonal so that no earlier update can break the tie.
# The later-offset row b is scaled by 2^30 from column c + 1 on (and empty before c): the first maximum keeps row a as
# the pivot row and b + a as an ordinary row; taking b instead would turn row a into a + b and lose it below the rounding
# of b, which the componentwise backward check sees at row a.  Column c + 1 then pivots on row b at offset > 1024.
WIDE_C = 8
WIDE_VARIANTS = {"far": (1040,), "tie_warp": (3, 1026), "tie_cross": (40, 1030)}
TIE = 16.0


def f4_wide(variant):
    rng = np.random.default_rng(40000 + len(variant))
    n, c = WIDE_N, WIDE_C
    # the orientation of a band after RCM is RCM's choice: build the pattern so that the permuted band is the lower one
    for offsets in (range(-2, WIDE_KL + 1), range(-WIDE_KL, 3)):
        rows, cols = _entries(n, offsets)
        case = _scrambled("F4-" + variant, n, rows, cols, np.zeros(rows.size), np.random.default_rng(4))
        if case.kl >= WIDE_KL:
            break
    assert case.kl > SLU_THREADS, case
    i, j = case.iperm[case.rowval], case.iperm[case.cols]     # band coordinates of every stored entry
    v = rng.standard_normal(i.size)
    offs = WIDE_VARIANTS[variant]
    col_c = j == c
    assert all(np.count_nonzero(col_c & (i == c + p)) == 1 for p in offs), (case, offs)
    v[col_c & (i < c)] = 0.0
    if variant == "far":
        v[col_c & (i >= c)] *= 2.0 ** -30
        v[col_c & (i == c + offs[0])] = TIE
    else:
        v[col_c & (i > c)] = np.clip(v[col_c & (i > c)], -4.0, 4.0)
        v[col_c & (i == c)] = 0.5
        b = c + offs[1]
        v[col_c & (i == c + offs[0])] = TIE
        v[col_c & (i == b)] = -TIE
        v[(i == b) & (j < c)] = 0.0
    big = (i == c + offs[-1]) & (j > c) if variant != "far" else np.zeros(i.size, dtype=bool)
    # strict column dominance everywhere else (the big row excluded, so that it pivots at column c + 1)
    diag = (i == j) & (j != c)
    dsum = np.bincount(j[~diag & ~big], weights=np.abs(v[~diag & ~big]), minlength=n)
    v[diag] = (dsum[j[diag]] + 1.0) * np.sign(rng.standard_normal(int(diag.sum())))
    v[big] *= BIG_ROW
    case.vals = v
    return case


def brusselator_case(nls, ctx, N):
    dp = nls._DeviceProblem(ctx, nls.NonlinearProblem(nls.Brusselator2D(N), None, (3.4, 1.0, 10.0), ctx=ctx))
    sj = nls.SparseJacobian(dp)
    nz = sj.fill(dp.u0(0)).to_host()
    cols = np.repeat(np.arange(dp.n), np.diff(sj.colptr))
    return Case("F6", dp.n, sj.rowval - 1, cols, nz)


def f1_cases():
    return [(kl, ku, n) for kl, ku in [(1, 1), (3, 7), (7, 3), (40, 40), (100, 5), (5, 100)] for n in (2, 31, 257, 1000, 3001) if kl < n]


SMALL_CASES = {"F2-n31": lambda: f2_no_diagonal(31), "F2-n257": lambda: f2_no_diagonal(257), "F2-n1000": lambda: f2_no_diagonal(1000, k=4, shift=9),
               "F3-n600": lambda: f3_disconnected(600), "F3-n2000": lambda: f3_disconnected(2000),
               "F5-diag-n1000": lambda: f5_diagonal(1000), "F5-n1": lambda: f5_diagonal(1)}
SMALL_CASES.update({"F1-kl%d-ku%d-n%d" % t: (lambda t=t: f1_band(*t)) for t in f1_cases()})


# ------------------------------------------------------------------------------------------------ LAPACK reference
class BandRef:
    """dgbtrf / dgbtrs on the RCM band of `case`, and |L|, |U| of P A_p = L U (A_p = A[perm][:, perm])."""

    def __init__(self, case, vals=None):
        self.case, n, kl, ku = case, case.n, case.kl, case.ku
        self.lu, self.ipiv, self.info = lapack.dgbtrf(case.band_array(vals), kl, ku)
        self.Ap = case.csr(vals)[case.perm][:, case.perm].tocsr()
        self.w = 3 * (2 * kl + ku + 1)
        kv = kl + ku
        piv = self.ipiv              # SciPy returns LAPACK's pivots 0-based
        self.swaps = int(np.count_nonzero(piv != np.arange(n)))
        self.max_offset = int((piv - np.arange(n)).max())
        if self.info != 0:
            return
        # row p of A_p ends at row m[p] of P A_p; the multipliers of column j are moved by the interchanges of later columns
        m = np.arange(n)
        Lr, Lc, Lv = [np.arange(n)], [np.arange(n)], [np.ones(n)]
        for j in range(n - 1, -1, -1):
            km = min(kl, n - 1 - j)
            if km:
                Lr.append(m[j + 1:j + 1 + km].copy())
                Lc.append(np.full(km, j))
                Lv.append(self.lu[kv + 1:kv + 1 + km, j])
            p = piv[j]
            m[j], m[p] = m[p], m[j]
        self.m = m
        self.L = sp.csr_matrix((np.concatenate(Lv), (np.concatenate(Lr), np.concatenate(Lc))), shape=(n, n))
        r, c = [], []
        for d in range(kv + 1):   # U[j - d, j] = lu[kv - d, j]
            j = np.arange(d, n)
            r.append(j - d)
            c.append(j)
        r, c = np.concatenate(r), np.concatenate(c)
        self.U = sp.csr_matrix((self.lu[kv - (c - r), c], (r, c)), shape=(n, n))
        self.absL, self.absU = abs(self.L), abs(self.U)
        self._ainv = None

    def solve(self, b):
        """LAPACK's solution of A x = b, in the original order."""
        x, info = lapack.dgbtrs(self.lu, self.case.kl, self.case.ku, b[self.case.perm].reshape(-1, 1), self.ipiv)
        assert info == 0
        out = np.empty_like(b)
        out[self.case.perm] = x[:, 0]
        return out

    def lux(self, y):
        """P^T |L| |U| y (in the order of A_p)."""
        return (self.absL @ (self.absU @ y))[self.m]

    def abs_inv(self):
        if self._ainv is None:
            import torch
            A = self.Ap.toarray()
            rmax = np.abs(A).max(axis=1)
            s = 2.0 ** -np.round(np.log2(np.where(rmax > 0, rmax, 1.0)))   # exact row equilibration: A^-1 = (S A)^-1 S
            Ainv = torch.linalg.inv(torch.tensor(s[:, None] * A, device="cuda")).cpu().numpy() * s[None, :]
            self._ainv = np.abs(Ainv)
        return self._ainv

    def check(self, b, x, forward=True):
        """Backward and forward checks of a device solution x of A x = b (original order)."""
        p = self.case.perm
        xp, bp = x[p], b[p]
        assert np.all(np.isfinite(xp)), self.case
        A = self.Ap
        prod = A.data.astype(np.longdouble) * xp.astype(np.longdouble)[A.indices]
        rowsum = np.zeros(self.case.n, dtype=np.longdouble)
        nonempty = np.diff(A.indptr) > 0
        rowsum[nonempty] = np.add.reduceat(prod, A.indptr[:-1][nonempty])
        r = np.abs((bp.astype(np.longdouble) - rowsum).astype(np.float64))
        g = gamma(self.w)
        bound = 2.0 * g * self.lux(np.abs(xp))
        bad = np.flatnonzero(r > bound)
        assert bad.size == 0, "%r: backward check fails at %d rows, e.g. row %d: |r| = %.3e > %.3e" % (self.case, bad.size, bad[0], r[bad[0]], bound[bad[0]])
        if not forward:
            return
        xl = self.solve(b)[p]
        fb = 2.0 * (self.abs_inv() @ (g * self.lux(np.maximum(np.abs(xp), np.abs(xl)))))
        d = np.abs(xp - xl)
        bad = np.flatnonzero(d > fb)
        assert bad.size == 0, "%r: forward check fails at %d entries, e.g. %d: %.3e > %.3e" % (self.case, bad.size, bad[0], d[bad[0]], fb[bad[0]])


def right_hand_sides(case, rng):
    n = case.n
    spread = np.where(rng.random(n) < 0.5, -1.0, 1.0) * 10.0 ** rng.uniform(-6.0, 6.0, n)
    return [rng.standard_normal(n), spread, case.csr() @ rng.standard_normal(n)]


def _bits(x):
    return np.ascontiguousarray(x).view(np.uint64)


# ------------------------------------------------------------------------------------------------ host-side references
def test_references_reproduce_superlu_and_the_families_pivot():
    """The restated RCM + LAPACK band solve reproduce SuperLU, and every pivoting family does pivot (so the device
    tests exercise the interchange, the fill up to kl + ku super-diagonals and the strided pivot search)."""
    import scipy.sparse.linalg as spla
    rng = np.random.default_rng(7)
    cases = [SMALL_CASES[k]() for k in SMALL_CASES] + [f4_wide(v) for v in WIDE_VARIANTS]
    for case in cases:
        ref = BandRef(case)
        assert ref.info == 0, case
        if case.n <= 2200:   # the factors the bounds are built from do reproduce P A_p = L U
            LU = (ref.L @ ref.U).toarray()[ref.m]
            assert np.all(np.abs(LU - ref.Ap.toarray()) <= gamma(ref.w) * (ref.absL @ ref.absU).toarray()[ref.m]), case
        A = case.csr().tocsc()
        lu = spla.splu(A)
        Ad = A.toarray()
        kappa = np.linalg.cond(Ad, np.inf)
        for b in right_hand_sides(case, rng):
            x, xs = ref.solve(b), lu.solve(b)
            assert np.abs(x - xs).max() <= 1e3 * U * kappa * np.abs(xs).max(), case
        if case.name in ("F1", "F2", "F3") and case.n >= 31:
            assert ref.swaps >= 0.3 * case.n, (case, ref.swaps)
        if case.name.startswith("F4"):
            assert ref.max_offset > SLU_THREADS, (case, ref.max_offset)
    # the pattern regimes the issue lists are all reached
    byname = {k: SMALL_CASES[k]() for k in ("F2-n31", "F3-n600", "F5-diag-n1000", "F5-n1", "F1-kl100-ku5-n1000", "F1-kl5-ku100-n1000")}
    assert byname["F5-diag-n1000"].kl == byname["F5-diag-n1000"].ku == 0 and byname["F5-n1"].n == 1
    assert byname["F1-kl100-ku5-n1000"].kl != byname["F1-kl100-ku5-n1000"].ku
    f2 = byname["F2-n31"]
    assert not np.any(f2.rowval == f2.cols)                                   # no structural diagonal
    f3 = byname["F3-n600"]
    ncomp = sp.csgraph.connected_components(f3.csr(), directed=False)[0]
    assert ncomp > 20 and np.any(np.bincount(f3.cols, minlength=f3.n) == 1)   # many components, isolated vertices among them


def test_rcm_restatement_on_a_path_and_a_star():
    """Hand-checkable orderings: a scrambled path is laid out end to end (bandwidth 1), and a star's centre comes last
    in the reversed order, after the leaves sorted by index."""
    n = 9
    q = np.array([4, 7, 0, 8, 2, 5, 1, 6, 3])
    rows, cols = q[:-1], q[1:]
    rows, cols = np.r_[rows, cols, np.arange(n)], np.r_[cols, rows, np.arange(n)]
    case = Case("path", n, rows, cols, np.ones(rows.size))
    assert (case.kl, case.ku) == (1, 1)
    assert list(case.perm) in (list(q), list(q[::-1]))
    leaves = np.arange(1, n)
    rows, cols = np.r_[leaves, np.zeros(n - 1, dtype=int)], np.r_[np.zeros(n - 1, dtype=int), leaves]
    star = Case("star", n, rows, cols, np.ones(rows.size))
    # root: vertex 0 has eccentricity 1, its last level (the leaves) gives leaf 1 with eccentricity 2 -> root 1
    assert list(star.perm) == list(reversed([1, 0, 2, 3, 4, 5, 6, 7, 8]))


# ------------------------------------------------------------------------------------------------ device: factor + solve
def _solve(nls, ctx, lu, b):
    return lu.solve(ctx.to_device(b)).to_host()


def check_factor_and_solves(nls, ctx, case, rng):
    ref = BandRef(case)
    lu = nls.SparseBandLU(ctx, case.n, case.colptr + 1, case.rowval + 1, 1)
    assert lu.bandwidth() == (case.kl, case.ku), case
    nz = ctx.to_device(case.vals)
    assert lu.factor(nz) == 0 and ref.info == 0, case
    rhs = right_hand_sides(case, rng)
    xs = []
    for b in rhs:
        x = _solve(nls, ctx, lu, b)
        ref.check(b, x)
        xs.append(x)
    # determinism: a second solve, an in-place solve, a re-factored handle and a fresh 0-based handle give the same bits
    b = rhs[0]
    assert np.array_equal(_bits(_solve(nls, ctx, lu, b)), _bits(xs[0]))
    db = ctx.to_device(b)
    assert np.array_equal(_bits(lu.solve(db, x=db).to_host()), _bits(xs[0]))
    other = case.vals * (1.0 + 0.5 * rng.standard_normal(case.vals.size))
    assert lu.factor(ctx.to_device(other)) == 0
    xo = _solve(nls, ctx, lu, b)
    BandRef(case, other).check(b, xo, forward=False)
    assert lu.factor(nz) == 0
    assert np.array_equal(_bits(_solve(nls, ctx, lu, b)), _bits(xs[0]))
    lu0 = nls.SparseBandLU(ctx, case.n, case.colptr, case.rowval, 0)
    assert lu0.bandwidth() == (case.kl, case.ku) and lu0.factor(nz) == 0
    assert np.array_equal(_bits(_solve(nls, ctx, lu0, rhs[1])), _bits(xs[1]))
    return lu, ref


def check_singular(nls, ctx, case, lu, columns, rows):
    """A zeroed column c stays exactly zero under every earlier update: info is iperm[c] + 1, as in LAPACK.  A zeroed row
    stays exactly zero too, so some pivot is exactly zero: info > 0 for both."""
    for c in columns:
        v = case.zeroed(column=c)
        info = lu.factor(ctx.to_device(v))
        assert info == case.iperm[c] + 1 == BandRef(case, v).info, (case, c, info)
    for r in rows:
        v = case.zeroed(row=r)
        assert lu.factor(ctx.to_device(v)) > 0 and BandRef(case, v).info > 0, (case, r)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SMALL_CASES))
def test_band_lu_families(nls, ctx, name):
    case = SMALL_CASES[name]()
    rng = np.random.default_rng(len(name) * 7919 + case.n)
    lu, ref = check_factor_and_solves(nls, ctx, case, rng)
    cols = sorted({0, case.n // 2, case.n - 1, int(case.perm[0]), int(case.perm[-1])})
    check_singular(nls, ctx, case, lu, cols, [case.n // 3])


@pytest.mark.gpu
@pytest.mark.parametrize("variant", list(WIDE_VARIANTS))
def test_band_lu_wide_band_pivots_past_the_thread_count(nls, ctx, variant):
    """kl = 1040 > 1024 threads: the pivot search takes a thread's second item, and the interchange, the fill, the
    multiplier scaling and both triangular sweeps run past one row per thread."""
    case = f4_wide(variant)
    assert case.kl > SLU_THREADS
    lu, ref = check_factor_and_solves(nls, ctx, case, np.random.default_rng(41))
    assert ref.max_offset > SLU_THREADS
    check_singular(nls, ctx, case, lu, [int(case.perm[WIDE_C + 30])], [])


@pytest.mark.gpu
def test_band_lu_brusselator_2d_n64(nls, ctx):
    """The size the route is meant for: n = 8192."""
    case = brusselator_case(nls, ctx, 64)
    assert case.n == 8192
    check_factor_and_solves(nls, ctx, case, np.random.default_rng(64))


# ------------------------------------------------------------------------------------------------ sparse.cu on general patterns
def general_pattern(n, rng):
    """Random CSC pattern with empty rows and columns and one dense row of 100-300 columns (> 64 colours)."""
    if n == 1:
        return sp.csc_matrix(np.array([[rng.standard_normal()]]))
    per_col = rng.integers(0, 6, n)
    cols = np.repeat(np.arange(n), per_col)
    rows = rng.integers(0, n, cols.size)
    dense_row = int(rng.integers(0, n))
    dcols = rng.choice(n, size=min(n, int(rng.integers(100, 301))), replace=False)
    rows, cols = np.r_[rows, np.full(dcols.size, dense_row)], np.r_[cols, dcols]
    empty_r = rng.choice(n, size=max(1, n // 20), replace=False)
    empty_c = rng.choice(n, size=max(1, n // 20), replace=False)
    empty_r = empty_r[empty_r != dense_row]
    keep = ~np.isin(rows, empty_r) & ~np.isin(cols, empty_c)
    rows, cols = rows[keep], cols[keep]
    key = np.unique(rows * n + cols)
    rows, cols = key // n, key % n
    vals = rng.standard_normal(rows.size) * 10.0 ** rng.uniform(-3, 3, rows.size)
    A = sp.csc_matrix((vals, (rows, cols)), shape=(n, n))
    A.sort_indices()
    return A


def two_prod(a, b):
    """a * b = p + e exactly (Dekker, Veltkamp splitting); no overflow for the magnitudes used here."""
    def split(x):
        t = 134217729.0 * x
        hi = t - (t - x)
        return hi, x - hi
    p = a * b
    ah, al = split(a)
    bh, bl = split(b)
    e = ((ah * bh - p) + ah * bl + al * bh) + al * bl
    return p, e


def exact_sums(indptr, idx, data, x):
    """Correctly rounded sum of data[k] * x[idx[k]] over each segment of indptr."""
    p, e = two_prod(data, x[idx])
    return np.array([math.fsum(np.r_[p[a:b], e[a:b]]) for a, b in zip(indptr[:-1], indptr[1:])])


@pytest.mark.gpu
@pytest.mark.parametrize("base", [0, 1])
@pytest.mark.parametrize("n", [1, 255, 256, 257, 5000])
def test_sparse_jacobian_on_general_patterns(nls, ctx, po, n, base):
    import torch
    rng = np.random.default_rng(n * 2 + base)
    A = general_pattern(n, rng)
    colptr, rowval = (A.indptr + base).astype(np.int64), (A.indices + base).astype(np.int64)
    At = torch.tensor(A.toarray(), device="cuda")

    def JVP(Jv, v, u, _p):
        torch.as_tensor(Jv, device="cuda").copy_(At @ torch.as_tensor(v, device="cuda"))
        torch.cuda.synchronize()

    def F(du, u, _p):
        JVP(du, u, u, _p)

    f = nls.NonlinearFunction(F, jvp=JVP, n=n, jac_prototype=(colptr, rowval, base))
    dp = nls._DeviceProblem(ctx, nls.NonlinearProblem(f, np.zeros(n), None, ctx=ctx))
    cp, rv = dp.pattern(base)
    assert np.array_equal(cp, colptr) and np.array_equal(rv, rowval)
    # colourings: bit-exact against the C oracle in both orders, and valid (columns sharing a row never share a colour)
    for order in (nls.abi.ORDER_NATURAL, nls.abi.ORDER_LARGEST_FIRST):
        colors, nc = nls.coloring_column(n, colptr, rowval, base, order)
        oc, onc = po.coloring_column(n, colptr, rowval, base, order)
        assert nc == onc and np.array_equal(colors, oc), order
        assert colors.min() >= 1 and colors.max() == nc
        Ar = A.tocsr()
        for r in range(n):
            cs = colors[Ar.indices[Ar.indptr[r]:Ar.indptr[r + 1]]]
            assert np.unique(cs).size == cs.size, (order, r)
    if n >= 255:
        assert nc > 64                                     # the `forbidden` table of the colouring was resized
    sj = nls.SparseJacobian(dp, colptr, rowval, index_base=base)
    assert sj.ncolors == nc
    nz = sj.fill(ctx.to_device(rng.standard_normal(n)))
    assert np.array_equal(nz.to_host(), A.data)            # one product per compressed entry, every other term an exact zero
    # SpMV and SpMV^T against correctly rounded row / column sums
    Ar = A.tocsr()
    for _ in range(2):
        x = rng.standard_normal(n) * 10.0 ** rng.uniform(-2, 2, n)
        dx = ctx.to_device(x)
        for tr, M in ((False, Ar), (True, A)):
            y = sj.mul(nz, dx, transpose=tr).to_host()
            ex = exact_sums(M.indptr, M.indices, M.data, x)
            ln = np.diff(M.indptr)
            mag = np.abs(M).multiply(np.abs(x)[None, :]).sum(axis=1).A1 if not tr else np.abs(M).T.multiply(np.abs(x)[None, :]).sum(axis=1).A1
            assert np.all(np.abs(y - ex) <= gamma(np.maximum(ln, 1)) * mag), tr
            assert np.all(y[ln == 0] == 0.0), tr
    if n >= 255:
        assert np.any(np.diff(Ar.indptr) == 0) and np.any(np.diff(A.indptr) == 0)


# ------------------------------------------------------------------------------------------------ end to end
class _CubicProblem:
    """F(u) = A u + 0.1 u^3 - b with a dense Jacobian, for oracle/newton_numpy.solve."""

    def __init__(self, A, b):
        self.A, self.b = A, b

    def f(self, u):
        return self.A @ u + 0.1 * u ** 3 - self.b

    def jac(self, u):
        return self.A + np.diag(0.3 * u * u)


@pytest.mark.gpu
@pytest.mark.parametrize("family,with_jac", [("F1", True), ("F1", False), ("F2", True), ("F2", False)])
def test_newton_on_the_sparse_direct_route_vs_numpy(nls, ctx, family, with_jac):
    import torch
    from oracle import newton_numpy as nn
    n = 600
    case = f1_band(7, 3, n) if family == "F1" else f2_no_diagonal(n)
    rng = np.random.default_rng(601)
    # Newton from 0.05 away from the root converges in 4 (F1) or 6 (F2) steps.  F1's diagonal is shifted by +-4, which
    # leaves 96% of the Jacobian's columns non-dominant and 70 interchanges in its LU.  F2 keeps A's diagonal empty,
    # so the Jacobian's diagonal is 0.3 u^2 alone, and its LU interchanges rows in 455 of 600 columns.
    if family == "F1":
        on = case.rowval == case.cols
        case.vals[on] += 4.0 * np.where(rng.random(int(on.sum())) < 0.5, -1.0, 1.0)
        ustar = rng.standard_normal(n)
    else:
        ustar = np.where(rng.random(n) < 0.5, -1.0, 1.0) * (1.5 + 0.5 * rng.random(n))
    # the Jacobian A + 0.3 diag(u^2) needs the diagonal in its prototype even where A has none
    diag = np.arange(n)
    on_diag = case.rowval == case.cols
    rows, cols = np.r_[case.rowval, diag[~np.isin(diag, case.cols[on_diag])]], np.r_[case.cols, diag[~np.isin(diag, case.cols[on_diag])]]
    vals = np.r_[case.vals, np.zeros(rows.size - case.vals.size)]
    o = np.lexsort((rows, cols))
    rows, cols, vals = rows[o], cols[o], vals[o]
    colptr = np.r_[0, np.cumsum(np.bincount(cols, minlength=n))].astype(np.int64) + 1
    rowval = rows.astype(np.int64) + 1
    A = sp.csr_matrix((vals, (rows, cols)), shape=(n, n)).toarray()
    b = A @ ustar + 0.1 * ustar ** 3
    u0 = ustar + 0.05 * rng.standard_normal(n)
    At, bt = torch.tensor(A, device="cuda"), torch.tensor(b, device="cuda")
    rows_t, vals_t, isdiag_t = torch.tensor(rows, device="cuda"), torch.tensor(vals, device="cuda"), torch.tensor(rows == cols, device="cuda")

    def F(du, u, _p):
        u_t = torch.as_tensor(u, device="cuda")
        torch.as_tensor(du, device="cuda").copy_(At @ u_t + 0.1 * u_t ** 3 - bt)
        torch.cuda.synchronize()

    def JVP(Jv, v, u, _p):
        u_t, v_t = torch.as_tensor(u, device="cuda"), torch.as_tensor(v, device="cuda")
        torch.as_tensor(Jv, device="cuda").copy_(At @ v_t + 0.3 * u_t * u_t * v_t)
        torch.cuda.synchronize()

    def JAC(nz, u, _p):
        u_t = torch.as_tensor(u, device="cuda")
        torch.as_tensor(nz, device="cuda").copy_(vals_t + torch.where(isdiag_t, 0.3 * u_t[rows_t] ** 2, 0.0))
        torch.cuda.synchronize()

    f = nls.NonlinearFunction(F, jvp=JVP, n=n, jac=JAC if with_jac else None, jac_prototype=(colptr, rowval, 1))
    sol = nls.solve(nls.NonlinearProblem(f, u0, None, ctx=ctx), nls.NewtonRaphson(), abstol=1e-10)
    ref = nn.solve(_CubicProblem(A, b), u0, termination=nn.Termination(abstol=1e-10))
    s = sol.stats
    assert sol.retcode == ref["retcode"] == nls.ReturnCode.Success
    assert s.nsteps == ref["nsteps"] and s.nfactors == s.nsolve == s.nsteps, (s, ref["nsteps"])
    fn = np.array([t.fnorm_inf for t in sol.trace])
    # 1e-8 relative, down to the rounding of the residual evaluation itself (a few terms of size |A||u| + |b|)
    floor = 32 * U * np.max(np.abs(A) @ np.abs(ustar) + 0.1 * np.abs(ustar) ** 3 + np.abs(b))
    assert np.allclose(fn[:-1], np.array(ref["fnorm_inf"])[:-1], rtol=1e-8, atol=floor), (fn, ref["fnorm_inf"])
    u = sol.u.to_host() if hasattr(sol.u, "to_host") else np.asarray(sol.u)
    assert np.abs(u - ref["u"]).max() <= 1e-10 * max(1.0, np.abs(ref["u"]).max())
