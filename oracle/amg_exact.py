"""Exact restatements of the setup arithmetic of the device AMG (csrc/amg.cu) and rigorous bounds for what is not restated
exactly.  Test infrastructure only.

Everything here reads a hierarchy as the device exports it (CSR arrays with sorted columns) and recomputes one step from the
device's own inputs, so a check isolates that step from the rounding upstream of it:
  * `fma` is IEEE fused multiply-add, exact in integers and rounded once (CPython's int / int division is correctly rounded);
  * `galerkin_exact`, `at_exact`: the pair-list products in the order DESIGN.md §4i documents (for an output (i, c) the terms
    in ascending column of X; R = P' holds P's rows in ascending order), an fma fold from 0.0;
  * `tentative_exact`, `rho_exact`, `sa_p_exact`, `rs_p_exact`: T, the Gershgorin bound, SA's P and the Ruge-Stueben
    interpolation weights with the operations of the device, each one rounded as IEEE double arithmetic rounds it;
  * `galerkin_bound`, `sa_p_bound`, `rs_p_bound`, `Cycle`: componentwise first-order error bounds (u = 2^-53) for a value
    computed twice, by the device and by scipy / NumPy, in different orders.

The matrix families of tests/test_gpu_amg_general.py are here too, so the CPU suite can pin what the restatements predict."""
import math

import numpy as np
import scipy.linalg as sla
import scipy.sparse as sp

U = 2.0 ** -53


def fma(a, b, s):
    """round(a * b + s) with one rounding, for finite doubles."""
    na, da = a.as_integer_ratio()
    nb, db = b.as_integer_ratio()
    ns, ds = s.as_integer_ratio()
    num = na * nb * ds + ns * da * db
    if num == 0:   # IEEE: an exact zero sum is +0 unless both addends are zeros of one sign
        return 0.0 if (a != 0.0 and b != 0.0) else (a * b) + s
    return num / (da * db * ds)


def csr(M, ncols):
    """(data, indices, indptr) as exported -> scipy CSR with `ncols` columns (explicit zeros kept)."""
    val, col, rowptr = M
    return sp.csr_matrix((np.asarray(val), np.asarray(col), np.asarray(rowptr)), shape=(len(rowptr) - 1, ncols))


def rows_of(M):
    return np.repeat(np.arange(M.shape[0]), np.diff(M.indptr))


def ones(M):
    return sp.csr_matrix((np.ones(M.nnz), M.indices, M.indptr), shape=M.shape)


def _fold_product(X, Y):
    """Z = X Y as the device's pair-list product computes it: Z's sorted structural pattern and, per entry, the fma fold over
    its terms in ascending X column.  X, Y scipy CSR with sorted indices; returns a dict-of-rows (list of {col: value})."""
    xv, xc, xp = X.data.tolist(), X.indices.tolist(), X.indptr.tolist()
    yv, yc, yp = Y.data.tolist(), Y.indices.tolist(), Y.indptr.tolist()
    out = []
    for i in range(X.shape[0]):
        acc = {}
        for q in range(xp[i], xp[i + 1]):
            a, j = xv[q], xc[q]
            for t in range(yp[j], yp[j + 1]):
                c = yc[t]
                acc[c] = fma(a, yv[t], acc.get(c, 0.0))
        out.append(acc)
    return out


def _to_csr(rows, ncols):
    indptr = np.zeros(len(rows) + 1, dtype=np.int64)
    indptr[1:] = np.cumsum([len(r) for r in rows])
    cols = np.fromiter((c for r in rows for c in sorted(r)), dtype=np.int64, count=int(indptr[-1]))
    vals = np.fromiter((r[c] for r in rows for c in sorted(r)), dtype=np.float64, count=int(indptr[-1]))
    return sp.csr_matrix((vals, cols, indptr), shape=(len(rows), ncols))


def galerkin_exact(A, P):
    """A_{l+1} = R (A P) bit for bit: A P by the fold in ascending A column, then R (A P) with R = P' (each R row lists P's
    rows in ascending order) by the fold in ascending P row.  Returns (A P, A_{l+1}) as CSR."""
    AP = _to_csr(_fold_product(A, P), P.shape[1])
    R = P.T.tocsr()
    R.sort_indices()
    return AP, _to_csr(_fold_product(R, AP), P.shape[1])


def product_terms(X, Y):
    """The largest number of terms of one entry of X Y (structural)."""
    Z = ones(X) @ ones(Y)
    return int(Z.data.max()) if Z.nnz else 0


def at_exact(A, T):
    """A T on its structural pattern, the fold in ascending A column."""
    return _to_csr(_fold_product(A, T), T.shape[1])


def tentative_exact(agg, b):
    """T's values and the next candidate: ||b on aggregate a|| = sqrt of the member-order sum of separately rounded b_i^2,
    T_i = b_i / ||b on agg_i||.  agg[i] = -1 for an isolated row."""
    na = int(agg.max()) + 1 if len(agg) else 0
    s = [0.0] * na
    for i, a in enumerate(agg.tolist()):
        if a >= 0:
            s[a] = s[a] + b[i] * b[i]
    nrm = [math.sqrt(x) for x in s]
    tval = [b[i] / nrm[a] for i, a in enumerate(agg.tolist()) if a >= 0]
    return np.array(tval), np.array(nrm)


def rho_exact(A):
    """max_i (sequential sum of |a_ij| in column order) / |a_ii|."""
    v, p, c = A.data.tolist(), A.indptr.tolist(), A.indices.tolist()
    best = 0.0
    for i in range(A.shape[0]):
        s, d = 0.0, None
        for q in range(p[i], p[i + 1]):
            s = s + abs(v[q])
            if c[q] == i:
                d = v[q]
        best = max(best, s / abs(d))
    return best


def sa_p_exact(A, T, AT, smooth_omega):
    """P on A T's pattern: fma(-(omega_P / rho) * (1 / a_ii), (A T)_q, T_q or 0)."""
    rho = rho_exact(A)
    diag = A.diagonal().tolist()
    tcol = {i: int(T.indices[T.indptr[i]]) for i in range(T.shape[0]) if T.indptr[i + 1] > T.indptr[i]}
    tval = {i: float(T.data[T.indptr[i]]) for i in tcol}
    out = np.empty(AT.nnz)
    w = smooth_omega / rho
    for i in range(AT.shape[0]):
        c = w * (1.0 / diag[i])
        for q in range(AT.indptr[i], AT.indptr[i + 1]):
            t = tval[i] if tcol.get(i, -1) == AT.indices[q] else 0.0
            out[q] = fma(-c, float(AT.data[q]), t)
    return out


def rs_p_exact(A, P, cf):
    """Direct interpolation weights as the device computes them (one row at a time, no fma): C rows hold 1.0; an F row's
    an / ap sum its negative / positive off-diagonals in column order, sn / sp its interpolatory entries; d = a_ii, lumped
    with ap when sp == 0; p = -((alpha or beta) * a_ij) / d."""
    cpts = np.flatnonzero(cf)
    av, ac, apt = A.data.tolist(), A.indices.tolist(), A.indptr.tolist()
    out = np.empty(P.nnz)
    for i in range(A.shape[0]):
        p0, p1 = int(P.indptr[i]), int(P.indptr[i + 1])
        if p1 == p0:
            continue
        if cf[i]:
            out[p0] = 1.0
            continue
        row = {ac[q]: av[q] for q in range(apt[i], apt[i + 1])}
        an = ap = sn = spos = 0.0
        for q in range(apt[i], apt[i + 1]):
            if ac[q] == i:
                continue
            v = av[q]
            if v < 0.0:
                an = an + v
            elif v > 0.0:
                ap = ap + v
        vals = [row[int(cpts[c])] for c in P.indices[p0:p1]]
        for v in vals:
            if v < 0.0:
                sn = sn + v
            elif v > 0.0:
                spos = spos + v
        d = row[i]
        alpha = an / sn if sn != 0.0 else 0.0
        beta = 0.0
        if spos == 0.0:
            d = d + ap
        else:
            beta = ap / spos
        for k, v in enumerate(vals):
            out[p0 + k] = -((alpha if v < 0.0 else beta) * v) / d
    return out


def on_pattern(S, V):
    """V's values read at the positions of the sorted pattern S (zero where V has no entry)."""
    V = V.tocsr()
    V.sort_indices()
    m = max(S.shape[1], 1)
    ks = rows_of(S).astype(np.int64) * m + S.indices
    kv = rows_of(V).astype(np.int64) * m + V.indices
    out = np.zeros(S.nnz)
    pos = np.searchsorted(ks, kv)
    hit = (pos < len(ks)) & (ks[np.minimum(pos, len(ks) - 1)] == kv)
    out[pos[hit]] = V.data[hit]
    return out


def gamma(k):
    return k * U / (1.0 - k * U)


def galerkin_bound(A, P, pattern):
    """(scipy's R (A P) on `pattern`, the bound on |device - scipy| there).  Each side computes an A P entry with at most k1
    terms (|error| <= gamma(k1) |A| |P|) and an R (A P) entry with at most k2 (|error| <= gamma(k2) |R| |A P^|), so each is
    within (gamma(k1) + gamma(k2) (1 + gamma(k1))) |P|' |A| |P| of the exact product and the two within twice that; 2.2 (k1 + k2) u
    exceeds it while (k1 + k2) u < 0.04."""
    k1 = product_terms(A, P)
    k2 = product_terms(P.T.tocsr(), ones(A) @ ones(P))
    assert (k1 + k2) * U < 0.04
    ref = on_pattern(pattern, P.T @ (A @ P))
    mag = on_pattern(pattern, abs(P).T @ (abs(A) @ abs(P)))
    return ref, 2.2 * (k1 + k2) * U * mag


def sa_p_bound(A, T, pattern, smooth_omega):
    """(P = T - (omega_P / rho) D^-1 A T by scipy on `pattern`, the bound on |device - scipy|).  A T: gamma(kt) |A| |T| per side;
    rho a sum of at most m terms and one division (relative gamma(m)), c = (omega_P / rho) (1 / a_ii) three more roundings,
    the fma one (NumPy: a product and a difference, two): per side (gamma(kt) + gamma(m + 5)) |c| |A| |T| + 2 u |P|, twice that
    between the two; 2.2 covers the second-order terms."""
    kt = product_terms(A, T)
    m = int(np.diff(A.indptr).max())
    rho = float((np.asarray(abs(A).sum(axis=1)).ravel() / np.abs(A.diagonal())).max())
    c = smooth_omega / rho / A.diagonal()
    AT = on_pattern(pattern, A @ T)
    Tp = on_pattern(pattern, T)
    ref = Tp - np.repeat(c, np.diff(pattern.indptr)) * AT
    mag = np.repeat(np.abs(c), np.diff(pattern.indptr)) * on_pattern(pattern, abs(A) @ abs(T))
    return ref, 2.2 * ((kt + m + 5) * U * mag + 2 * U * np.abs(ref))


def rs_p_bound(A, P, cf):
    """(the restated direct interpolation on the device's A and P pattern, the bound on |device - restatement|).  alpha is a
    ratio of two same-signed sums of at most m terms (relative gamma(2 m + 1)); the product, the division and the negation
    add two roundings; d = a_ii + ap (when lumped) is a mixed-sign sum whose absolute error is at most gamma(m) (|a_ii| + ap),
    relative to d that times (|a_ii| + ap) / |d|.  Per side rel = gamma(2 m + 3) + gamma(m) (|a_ii| + ap) / |d|, twice between
    the two, 2.2 with the second order."""
    n = A.shape[0]
    rows, cols, v = rows_of(A), A.indices, A.data
    off = cols != rows
    m = int(np.diff(A.indptr).max())
    diag = A.diagonal()
    an, ap, sn, spos = (np.zeros(n) for _ in range(4))
    np.add.at(an, rows[off & (v < 0)], v[off & (v < 0)])
    np.add.at(ap, rows[off & (v > 0)], v[off & (v > 0)])
    cpts = np.flatnonzero(cf)
    pr = rows_of(P)
    pv = A[pr, cpts[P.indices]].A1 if P.nnz else np.zeros(0)
    F = ~cf[pr]
    np.add.at(sn, pr[F & (pv < 0)], pv[F & (pv < 0)])
    np.add.at(spos, pr[F & (pv > 0)], pv[F & (pv > 0)])
    alpha = np.divide(an, sn, out=np.zeros(n), where=sn != 0)
    beta = np.divide(ap, spos, out=np.zeros(n), where=spos != 0)
    lump = spos == 0
    d = np.where(lump, diag + ap, diag)
    w = np.where(pv < 0, alpha[pr], beta[pr])
    ref = np.where(F, -w * pv / d[pr], 1.0)
    scale = np.where(lump, np.abs(diag) + ap, np.abs(diag)) / np.abs(d)
    rel = gamma(2 * m + 3) + gamma(m) * scale[pr]
    return ref, np.where(F, 2.2 * rel * np.abs(ref), 0.0)


class Cycle:
    """One V(pre, post) cycle from x = 0 on a hierarchy given as its matrices (A_l, P_l with R_l = P_l', and the coarsest A_c),
    evaluated in NumPy together with a componentwise bound e on |computed - exact| that holds for the device's evaluation and
    for this one alike (so the two differ by at most 2 e; `bound(b)` returns 2.2 e for the second order).

    Rules, first order in u, for x^ = x + dx with |dx| <= e: y = M x with rows of at most k terms gives
    e_y = |M| e_x + gamma(k) |M| |x|; an elementwise product or sum adds u |result| per rounding (four covers both evaluations of
    the damped Jacobi update); the coarsest solve with an inverse X^ from LU with partial pivoting,
    |X^ - A_c^-1| <= gamma(3 n_c) |A_c^-1| |L| |U| |X^| (Higham, Accuracy and Stability, §14.3), plus its GEMV gamma(n_c) |X| |b|;
    |L| |U| are those of scipy's LU of A_c, the same partial-pivoting rule as getrf."""

    def __init__(self, As, Ps, Ac, omega=2.0 / 3.0, pre=1, post=1):
        self.As, self.Ps, self.omega, self.pre, self.post = As, Ps, omega, pre, post
        self.Ac = Ac.toarray()
        nc = self.Ac.shape[0]
        self.X = np.linalg.inv(self.Ac)
        Pm, L, Uf = sla.lu(self.Ac)
        absX = np.abs(self.X)
        self.Xerr = gamma(3 * nc) * (absX @ (np.abs(L) @ np.abs(Uf)) @ absX)
        self.nc = nc
        self.k = [int(np.diff(A.indptr).max()) for A in As]
        self.kp = [int(np.diff(P.indptr).max()) if P.nnz else 0 for P in Ps]
        self.kr = [int(np.diff(P.T.tocsr().indptr).max()) if P.nnz else 0 for P in Ps]

    def _apply(self, b, eb, l):
        if l == len(self.As):
            x = self.X @ b
            e = np.abs(self.X) @ eb + self.Xerr @ np.abs(b) + gamma(self.nc) * (np.abs(self.X) @ np.abs(b))
            return x, e
        A, P, k = self.As[l], self.Ps[l], self.k[l]
        aA, aP = abs(A), abs(P)
        dinv = 1.0 / A.diagonal()
        wd = self.omega * dinv
        col = (lambda v: v[:, None]) if b.ndim == 2 else (lambda v: v)  # noqa: E731
        x, e = np.zeros_like(b), np.zeros_like(b)

        def sweep(x, e):
            Ax = A @ x
            res = b - Ax
            eres = eb + aA @ e + gamma(k) * (aA @ np.abs(x)) + U * np.abs(res)
            y = x + col(wd) * res
            return y, e + col(np.abs(wd)) * (eres + 2 * U * np.abs(res)) + 4 * U * np.abs(y)

        for _ in range(self.pre):
            x, e = sweep(x, e)
        Ax = A @ x
        r = b - Ax
        er = eb + aA @ e + gamma(k) * (aA @ np.abs(x)) + U * np.abs(r)
        bc = P.T @ r
        ebc = aP.T @ er + gamma(self.kr[l]) * (aP.T @ np.abs(r))
        xc, exc = self._apply(bc, ebc, l + 1)
        x = x + P @ xc
        e = e + aP @ exc + gamma(self.kp[l]) * (aP @ np.abs(xc)) + U * np.abs(x)
        for _ in range(self.post):
            x, e = sweep(x, e)
        return x, e

    def __call__(self, b):
        return self._apply(b, np.zeros_like(b), 0)[0]

    def bound(self, b):
        """(the cycle of b, 2.2 e)."""
        x, e = self._apply(b, np.zeros_like(b), 0)
        return x, 2.2 * e


# ---------------------------------------------------------------- matrix families (scipy CSR, sorted, explicit zeros kept)
def _sorted(A):
    A = A.tocsr()
    A.sort_indices()
    return A


def one_sided(n, seed):
    """The diagonal and a_{i,i+1} only: every strong connection of the symmetric SA graph points one way."""
    rng = np.random.default_rng(seed)
    return _sorted(sp.diags([4.0 + rng.random(n), -(0.5 + rng.random(max(n - 1, 0)))], [0, 1], shape=(n, n)))


def laplacian_components(n, seed, ncomp=4, singletons=5):
    """Graph Laplacians of `ncomp` random connected-ish components plus `singletons` isolated nodes, + 0.1 I."""
    rng = np.random.default_rng(seed)
    sizes = np.diff(np.linspace(0, n - singletons, ncomp + 1).astype(int))
    blocks = []
    for m in sizes:
        W = sp.random(m, m, density=min(1.0, 4.0 / m), random_state=rng, data_rvs=lambda k: rng.uniform(0.1, 2.0, k))
        W = W + sp.diags(rng.uniform(0.1, 2.0, m - 1), 1, shape=(m, m))   # a path keeps the component connected
        W = ((W + W.T) * 0.5).tolil()
        W.setdiag(0.0)
        W = W.tocsr()
        W.eliminate_zeros()
        blocks.append(sp.diags(np.asarray(W.sum(axis=1)).ravel()) - W)
    blocks.append(sp.csr_matrix((singletons, singletons)))
    L = sp.block_diag(blocks).tocsr()
    return _sorted(L + 0.1 * sp.identity(n) + sp.diags(np.zeros(n)))


def arrow(n, hub=1e-6):
    """A strong tridiagonal chain (2, -1) on nodes 1..n-1 plus a weak dense hub: row and column 0 hold |a_0j| = |a_j0| = hub
    (both signs) for every j, so the hub has no strong connection."""
    A = sp.diags([-np.ones(n - 1), 2.0 * np.ones(n), -np.ones(n - 1)], [-1, 0, 1], shape=(n, n), format="lil")
    s = np.where(np.arange(n) % 2 == 0, hub, -hub)
    A[0, 1:] = s[1:]
    A[1:, 0] = s[1:, None]
    return _sorted(A)


def star(n, seed):
    """A hub strongly coupled to every node, the leaves coupled only to it: every node is within distance 2 of every other."""
    rng = np.random.default_rng(seed)
    A = sp.lil_matrix((n, n))
    A.setdiag(2.0 + rng.random(n))
    A[0, 0] = 4.0          # small enough that every hub entry is strong: |a_0j| >= 0.5 > 0.08 sqrt(4 * 3)
    A[0, 1:] = -(0.5 + rng.random(n - 1))
    A[1:, 0] = -(0.5 + rng.random((n - 1, 1)))
    return _sorted(A)


def with_stored_zeros(A, seed, frac=0.05):
    """A with `frac` of its off-diagonal values set to 0.0, each kept as a structural entry."""
    A = A.copy().tocsr()
    rng = np.random.default_rng(seed)
    off = np.flatnonzero(A.indices != rows_of(A))
    A.data[rng.choice(off, size=max(1, int(frac * len(off))), replace=False)] = 0.0
    return A


def rows_scaled(A, seed, kmax=20):
    """Row i times 2^k_i, k_i uniform in [-kmax, kmax] (exact)."""
    rng = np.random.default_rng(seed)
    k = rng.integers(-kmax, kmax + 1, A.shape[0])
    return _sorted(sp.diags(np.ldexp(1.0, k)) @ A)


def banded(n, seed, width=2):
    """Random values of both signs in the band |i - j| <= width, 4 + U(0, 1) on the diagonal: a sparse matrix whose coarse levels
    stay banded (no fill), so n can be large at small cost."""
    rng = np.random.default_rng(seed)
    diags = [rng.standard_normal(n - abs(k)) for k in range(-width, width + 1)]
    diags[width] = 4.0 + rng.random(n)
    return _sorted(sp.diags(diags, list(range(-width, width + 1)), shape=(n, n)))
