"""Independent whole-array restatement (NumPy / scipy.sparse) of the smoothed-aggregation AMG of csrc/amg.cu, written from the
rules of DESIGN.md §4i, not from the CUDA: symmetric strength, the distance-2 maximal independent set, the two aggregation
passes, the tentative prolongator, its Jacobi smoothing with the Gershgorin bound, and the frozen-aggregate refresh.  The
Galerkin product and the V-cycle are those of the Ruge-Stueben restatement (oracle/amg_numpy.py).  Test infrastructure only.

Matrices are scipy CSR with sorted indices and every structural entry kept, as in amg_numpy: patterns are structural."""
import numpy as np
import scipy.sparse as sp

from oracle import amg_numpy as am

OUT, UNDECIDED, IN = 0, 1, 2


def hash32(i):
    """The node priority h(i): x ^= x>>16; x *= 0x7feb352d; x ^= x>>15; x *= 0x846ca68b; x ^= x>>16 (a bijection of uint32)."""
    x = np.asarray(i, dtype=np.uint32).copy()
    x ^= x >> np.uint32(16)
    x *= np.uint32(0x7FEB352D)
    x ^= x >> np.uint32(15)
    x *= np.uint32(0x846CA68B)
    x ^= x >> np.uint32(16)
    return x


def _one(M):
    return sp.csr_matrix((np.ones(M.nnz), M.indices, M.indptr), shape=M.shape)


def _on_pattern(S, V):
    """V's values at the positions of the (sorted, structural) pattern S, zero where V has no entry; V's pattern lies in S's."""
    V = V.tocsr()
    V.sort_indices()
    m = S.shape[1]
    ks = am._rows(S).astype(np.int64) * m + S.indices
    kv = am._rows(V).astype(np.int64) * m + V.indices
    out = np.zeros(S.nnz)
    out[np.searchsorted(ks, kv)] = V.data
    return sp.csr_matrix((out, S.indices.copy(), S.indptr.copy()), shape=S.shape)


def strength_graph(A, theta=0.08):
    """The symmetric strength graph (a 0/1 CSR without diagonal): j != i is strong for i when a_ij != 0 and
    |a_ij| >= theta sqrt(|a_ii| |a_jj|); (i, j) is an edge when either (i, j) or (j, i) is strong."""
    n = A.shape[0]
    rows, cols, v = am._rows(A), A.indices, A.data
    d = np.abs(A.diagonal())
    s = (cols != rows) & (v != 0.0) & (np.abs(v) >= theta * np.sqrt(d[rows] * d[cols]))
    S = sp.csr_matrix((np.ones(int(s.sum())), (rows[s], cols[s])), shape=(n, n))
    G = _one((S + S.T).tocsr())
    G.sort_indices()
    return G


def _nbr_max(G, x):
    """m[i] = max(x[i], max of x over i's neighbours)."""
    m = x.copy()
    has = np.diff(G.indptr) > 0
    if G.nnz:
        m[has] = np.maximum(m[has], np.maximum.reduceat(x[G.indices], G.indptr[:-1][has]))
    return m


def mis2(G):
    """Distance-2 maximal independent set: (state per node, rounds).  Each node carries (state, h) as one integer, IN >
    UNDECIDED > OUT; a round takes two max-propagations, then an undecided node that is its own distance-2 maximum becomes IN and
    one whose maximum is IN becomes OUT.  Isolated nodes start OUT."""
    n = G.shape[0]
    h = hash32(np.arange(n)).astype(np.uint64)
    iso = np.diff(G.indptr) == 0
    state = np.where(iso, OUT, UNDECIDED).astype(np.uint64)
    rounds = 0
    while (state == UNDECIDED).any():
        rounds += 1
        key = (state << np.uint64(32)) | h
        m2 = _nbr_max(G, _nbr_max(G, key))
        und = state == UNDECIDED
        state = np.where(und & (m2 == key), IN, np.where(und & ((m2 >> np.uint64(32)) == IN), OUT, state)).astype(np.uint64)
    return state.astype(np.int64), rounds


def _best_neighbour(G, ok, score):
    """For every node, the neighbour j with ok[j] of largest score[j] (-1 where there is none)."""
    r, c = am._rows(G), G.indices
    m = ok[c]
    r, c = r[m], c[m]
    order = np.lexsort((score[c], r))
    r, c = r[order], c[order]
    last = np.r_[r[1:] != r[:-1], True] if len(r) else np.zeros(0, dtype=bool)
    best = -np.ones(G.shape[0], dtype=np.int64)
    best[r[last]] = c[last]
    return best


def aggregate(G):
    """Aggregate number per node (-1: isolated), the number of aggregates, and the MIS states and rounds."""
    n = G.shape[0]
    state, rounds = mis2(G)
    root = state == IN
    rid = np.cumsum(root) - 1
    h = hash32(np.arange(n)).astype(np.int64)
    agg = np.where(root, rid, -1)
    b1 = _best_neighbour(G, root, h)                       # pass 1: the adjacent root of largest h
    agg1 = np.where(root, rid, np.where(b1 >= 0, rid[np.maximum(b1, 0)], -1))
    b2 = _best_neighbour(G, agg1 >= 0, h)                  # pass 2: the assigned neighbour of largest h
    agg = np.where(agg1 >= 0, agg1, np.where(b2 >= 0, agg1[np.maximum(b2, 0)], -1))
    return agg, int(root.sum()), state, rounds


def tentative(agg, na, b):
    """T (n x na, one entry b_i / ||b on the aggregate|| per aggregated row) and the next candidate (the aggregates' norms)."""
    n = len(agg)
    m = agg >= 0
    nrm = np.sqrt(np.bincount(agg[m], weights=b[m] * b[m], minlength=na))
    T = sp.csr_matrix((b[m] / nrm[agg[m]], (np.flatnonzero(m), agg[m])), shape=(n, na))
    T.sort_indices()
    return T, nrm


def rho(A):
    """The Gershgorin bound max_i sum_j |a_ij| / |a_ii| of D^-1 A."""
    return float((np.asarray(abs(A).sum(axis=1)).ravel() / np.abs(A.diagonal())).max())


def smoothed(A, T, smooth_omega=4.0 / 3.0):
    """P = T - (omega_P / rho) D^-1 A T on the structural pattern of A T (which holds T's: every row has a diagonal)."""
    S = (_one(A) @ _one(T)).tocsr()
    S.sort_indices()
    AT = _on_pattern(S, A @ T)
    Tp = _on_pattern(S, T)
    c = smooth_omega / rho(A) / A.diagonal()
    P = Tp.copy()
    P.data = Tp.data - np.repeat(c, np.diff(S.indptr)) * AT.data
    return P


class Hierarchy(am.Hierarchy):
    """levels[l] = dict(A, P, T, agg, state, G) for every level but the coarsest; coarse = the coarsest A.  cycle(b) as in
    amg_numpy (V(pre, post), damped Jacobi, the coarsest level's explicit inverse)."""

    def __init__(self, A, theta=0.08, omega=2.0 / 3.0, presweeps=1, postsweeps=1, max_levels=10, max_coarse=10, smooth_omega=4.0 / 3.0,
                 frozen=None):
        self.omega, self.pre, self.post, self.smooth_omega = omega, presweeps, postsweeps, smooth_omega
        self.levels = []
        A = A.tocsr()
        b = np.ones(A.shape[0])
        while True:
            l = len(self.levels)
            if frozen is not None:
                if l == len(frozen.levels):
                    break
                F = frozen.levels[l]
                G, agg, state, T = F["G"], F["agg"], F["state"], F["T"]
            else:
                if A.shape[0] <= max_coarse or l + 1 >= max_levels:
                    break
                G = strength_graph(A, theta)
                agg, na, state, _ = aggregate(G)
                if na == 0 or na == A.shape[0]:
                    break
                T, b = tentative(agg, na, b)
            P = smoothed(A, T, smooth_omega)
            self.levels.append(dict(A=A, P=P, T=T, agg=agg, state=state, G=G))
            A = am.galerkin(A, P)
        self.coarse = A
        self._coarse_inv = None

    def refresh(self, A0):
        """The same aggregates, T and patterns, every value recomputed from the new level-0 values."""
        return Hierarchy(A0, omega=self.omega, presweeps=self.pre, postsweeps=self.post, smooth_omega=self.smooth_omega, frozen=self)
