"""ILU(0) restated in NumPy, independently of the device code (csrc/ilu0.cu): level sets of the strictly lower / upper
patterns, row-wise IKJ incomplete LU with zero fill, and the two triangular sweeps.  Patterns are CSC (colptr, rowval) with
an explicit index base, as the C ABI takes them; packed factors are returned in that CSC order (L strictly below the
diagonal with an implied unit diagonal, U on and above it)."""
import numpy as np


def _rows(n, colptr, rowval, index_base):
    """Row i -> (columns ascending, CSC positions) as two int arrays."""
    colptr = np.asarray(colptr, dtype=np.int64) - index_base
    rowval = np.asarray(rowval, dtype=np.int64) - index_base
    cols = np.repeat(np.arange(n), np.diff(colptr))
    order = np.lexsort((cols, rowval))
    bounds = np.searchsorted(rowval[order], np.arange(n + 1))
    return [(cols[order[bounds[i]:bounds[i + 1]]], order[bounds[i]:bounds[i + 1]]) for i in range(n)]


def _diag(rows):
    d = []
    for i, (c, p) in enumerate(rows):
        hit = np.nonzero(c == i)[0]
        if len(hit) == 0:
            raise ValueError("row %d has no structural diagonal entry" % i)
        d.append(int(p[hit[0]]))
    return d


def levels(n, colptr, rowval, index_base=1):
    """Level of every row in the forward sweep (longest chain of strictly lower dependencies) and in the backward sweep."""
    rows = _rows(n, colptr, rowval, index_base)
    lo = np.zeros(n, dtype=np.int64)
    up = np.zeros(n, dtype=np.int64)
    for i in range(n):
        c = rows[i][0]
        dep = c[c < i]
        lo[i] = lo[dep].max() + 1 if len(dep) else 0
    for i in range(n - 1, -1, -1):
        c = rows[i][0]
        dep = c[c > i]
        up[i] = up[dep].max() + 1 if len(dep) else 0
    return lo, up


def level_counts(n, colptr, rowval, index_base=1):
    lo, up = levels(n, colptr, rowval, index_base)
    return int(lo.max()) + 1, int(up.max()) + 1


def ilu0(n, colptr, rowval, nzval, index_base=1):
    """Packed ILU(0) factors in CSC order and info (0, or the 1-based row of the first zero / non-finite pivot)."""
    rows = _rows(n, colptr, rowval, index_base)
    diag = _diag(rows)
    a = np.array(nzval, dtype=np.float64)
    where = [dict(zip(c.tolist(), p.tolist())) for c, p in rows]   # row -> {column: CSC position}
    info = 0
    for i in range(n):
        cols, pos = rows[i]
        for t in range(len(cols)):
            k = int(cols[t])
            if k >= i:
                break
            pk = int(pos[t])
            a[pk] = a[pk] / a[diag[k]]
            for j, pj in zip(cols[t + 1:].tolist(), pos[t + 1:].tolist()):
                q = where[k].get(j)
                if q is not None:
                    a[pj] = a[pj] - a[pk] * a[q]
        d = a[diag[i]]
        if info == 0 and (d == 0.0 or not np.isfinite(d)):
            info = i + 1
    return a, info


def solve(n, colptr, rowval, factors, b, index_base=1):
    """x = U^-1 L^-1 b from packed factors (unit lower L)."""
    rows = _rows(n, colptr, rowval, index_base)
    diag = _diag(rows)
    f = np.asarray(factors, dtype=np.float64)
    x = np.array(b, dtype=np.float64)
    for i in range(n):
        c, p = rows[i]
        m = c < i
        x[i] = x[i] - np.dot(f[p[m]], x[c[m]])
    for i in range(n - 1, -1, -1):
        c, p = rows[i]
        m = c > i
        x[i] = (x[i] - np.dot(f[p[m]], x[c[m]])) / f[diag[i]]
    return x


def dense_factors(n, colptr, rowval, factors, index_base=1):
    """(L, U) as dense matrices from packed factors."""
    colptr = np.asarray(colptr, dtype=np.int64) - index_base
    rowval = np.asarray(rowval, dtype=np.int64) - index_base
    cols = np.repeat(np.arange(n), np.diff(colptr))
    L = np.eye(n)
    U = np.zeros((n, n))
    low = rowval > cols
    L[rowval[low], cols[low]] = np.asarray(factors)[low]
    U[rowval[~low], cols[~low]] = np.asarray(factors)[~low]
    return L, U
