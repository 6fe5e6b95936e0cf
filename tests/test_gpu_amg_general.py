"""Both device AMG setups (csrc/amg.cu: Ruge-Stueben and smoothed aggregation) on general sparse matrices, through the device
sparse product they share.

Every family runs through both methods.  Structure (level sizes, every pattern of A_l and P_l, SA's T) is compared with the
restatements (oracle/amg_numpy.py, oracle/sa_numpy.py) exactly; values step by step from the device's own exported inputs, either
bit for bit against an exact restatement of the device arithmetic or within a componentwise bound derived for the operation
(oracle/amg_exact.py states each derivation).  No tolerance here is a tuned constant."""
import ctypes as C

import numpy as np
import pytest
import scipy.linalg as sla
import scipy.sparse as sp

from oracle import amg_exact as ax
from oracle import amg_numpy as am
from oracle import sa_numpy as sa
from test_amg_oracle import random_matrix
from test_gpu_amg import _csc_of

pytestmark = pytest.mark.gpu

METHODS = ("rs", "sa")

# name -> scipy CSR; every family runs through both methods
FAMILIES = {
    **{"random%d" % n: (lambda n=n: random_matrix(n, 11 + n)) for n in (1, 2, 9, 10, 11, 255, 256, 257, 4097)},
    "one_sided": lambda: ax.one_sided(300, 1),
    "laplacian_components": lambda: ax.laplacian_components(600, 2),
    "arrow": lambda: ax.arrow(2000),
    "star": lambda: ax.star(300, 3),
    "stored_zeros": lambda: ax.with_stored_zeros(random_matrix(800, 4), 4),
    "rows_scaled": lambda: ax.rows_scaled(random_matrix(800, 5), 5),
    # SA's level-0 transpose key reaches n^2 - 1, which needs 32 bits at n = 65536 and 33 at 65537 whatever the values; only
    # the diagonal's last columns reach the top bit.  A banded matrix crosses that boundary without the coarse-level fill of
    # a random graph
    "keywidth65536": lambda: ax.banded(65536, 6),
    "keywidth65537": lambda: ax.banded(65537, 7),
}
LARGE = {"keywidth65536", "keywidth65537"}
CASES = [(f, m) for f in FAMILIES for m in METHODS]
IDS = ["%s-%s" % c for c in CASES]
# small members: every value restated bit for bit (pure-Python fma folds)
EXACT = [c for c in CASES if c[0] not in ("random4097", "arrow") and c[0] not in LARGE]
# the form and scaling checks run on everything but the two largest
FORMS = [c for c in CASES if c[0] not in LARGE]

_cache = {}


def family(name):
    if name not in _cache:
        _cache[name] = FAMILIES[name]()
    return _cache[name]


def restate(method, A, **opts):
    return (sa.Hierarchy if method == "sa" else am.Hierarchy)(A, **opts)


def make(nls, ctx, method, A, base=1, **opts):
    cp, rv, nz = _csc_of(A, base)
    n = A.shape[0]
    h = nls.SparseAMG.smoothed_aggregation(ctx, n, cp, rv, base, **opts) if method == "sa" else nls.SparseAMG(ctx, n, cp, rv, base, **opts)
    return h, cp, rv, nz


def export(amg):
    """(sizes, [A_l], [P_l], [T_l]) as scipy CSR from the device."""
    ns, _ = amg.levels()
    As, Ps, Ts = [], [], []
    for l, n in enumerate(ns):
        lv = amg.level(l)
        As.append(ax.csr(lv["A"], n))
        if l + 1 < len(ns):
            Ps.append(ax.csr(lv["P"], ns[l + 1]))
            if lv.get("T") is not None:
                Ts.append(ax.csr(lv["T"], ns[l + 1]))
        else:
            assert lv["P"] is None and lv.get("T") is None
    return ns, As, Ps, Ts


def raw(amg):
    """Every exported array of the hierarchy, for bit comparisons."""
    ns, As, Ps, Ts = export(amg)
    return [a for M in As + Ps + Ts for a in (M.indptr, M.indices, M.data)]


def bits(x):
    return np.ascontiguousarray(x).view(np.uint8)


def same_bits(a, b):
    return len(a) == len(b) and all(x.dtype == y.dtype and np.array_equal(bits(x), bits(y)) for x, y in zip(a, b))


def same_pattern(M, R):
    return M.shape == R.shape and np.array_equal(M.indptr, R.indptr) and np.array_equal(M.indices, R.indices)


def within(got, ref, bound, what):
    err = np.abs(got - ref)
    bad = ~(err <= bound)
    assert not bad.any(), "%s: %d entries outside the bound, worst |d| = %g at bound %g" % (
        what, int(bad.sum()), err[bad].max(), bound[bad][np.argmax(err[bad])])


def check_values(method, ns, As, Ps, Ts, cfs=None, smooth_omega=4.0 / 3.0):
    """Every P_l and A_{l+1} from the device's A_l (and T_l, or the splitting cfs[l]) within the derived bounds."""
    for l in range(len(ns) - 1):
        A, P = As[l], Ps[l]
        if method == "sa":
            ref, bnd = ax.sa_p_bound(A, Ts[l], P, smooth_omega)
        else:
            ref, bnd = ax.rs_p_bound(A, P, cfs[l])
        within(P.data, ref, bnd, "P_%d" % l)
        ref, bnd = ax.galerkin_bound(A, P, As[l + 1])
        within(As[l + 1].data, ref, bnd, "A_%d" % (l + 1))


def check_cycle(amg, ctx, As, Ps, omega, pre, post, seed):
    b = np.random.default_rng(seed).standard_normal(As[0].shape[0])
    cyc = ax.Cycle(As[:-1], Ps, As[-1], omega, pre, post)
    ref, bnd = cyc.bound(b)
    x = amg.solve(ctx.to_device(b)).to_host()
    within(x, ref, bnd, "cycle")
    return b, x


def check_steps(method, ns, As, Ps, Ts, opts):
    """Each level's coarsening decided by the restatement's rules on the device's own A_l: the same P_l (and T_l) pattern."""
    for l in range(len(ns) - 1):
        Hl = restate(method, As[l], **{**opts, "max_levels": 2, "max_coarse": 1})
        assert Hl.sizes() == ns[l:l + 2], l
        assert same_pattern(Ps[l], Hl.levels[0]["P"]), l
        if method == "sa":
            assert same_pattern(Ts[l], Hl.levels[0]["T"]), l


def check_against_restatement(amg, ctx, method, H, A0, seed=1, opts=None, stepwise=False):
    """Structure exactly (sizes, nnz, every pattern; SA's T and the aggregates bit for bit), values within the bounds of
    check_values, one cycle within the bound of amg_exact.Cycle evaluated on the device's own hierarchy.  With `stepwise` the
    structure is compared level by level (check_steps) instead of against the whole restated hierarchy."""
    ns, As, Ps, Ts = export(amg)
    if stepwise:
        check_steps(method, ns, As, Ps, Ts, opts or {})
        check_values(method, ns, As, Ps, Ts, [am.split(M, am.strength(M, (opts or {}).get("theta", 0.25))) for M in As[:-1]]
                     if method == "rs" else None, (opts or {}).get("smooth_omega", 4.0 / 3.0))
        return check_cycle(amg, ctx, As, Ps, H.omega, H.pre, H.post, seed)
    assert ns == H.sizes()
    assert [M.nnz for M in As] == H.nnz()
    assert same_pattern(As[0], A0) and same_bits([As[0].data], [A0.data])      # level 0 is the caller's values, gathered
    for l in range(len(ns) - 1):
        Lo = H.levels[l]
        assert same_pattern(As[l], Lo["A"]), l
        assert same_pattern(Ps[l], Lo["P"]), l
        if method == "sa":
            assert same_pattern(Ts[l], Lo["T"]) and same_bits([Ts[l].data], [Lo["T"].data]), l
    assert same_pattern(As[-1], H.coarse)
    check_values(method, ns, As, Ps, Ts, [L.get("cf") for L in H.levels], getattr(H, "smooth_omega", 4.0 / 3.0))
    return check_cycle(amg, ctx, As, Ps, H.omega, H.pre, H.post, seed)


# ---------------------------------------------------------------------------------------------------------------- (a)
@pytest.mark.parametrize("fam,method", CASES, ids=IDS)
def test_hierarchy_against_the_restatement(nls, ctx, fam, method):
    A = family(fam)
    amg, cp, rv, nz = make(nls, ctx, method, A)
    assert amg.setup(ctx.to_device(nz)) == 0
    A0 = am.csr_of_csc(A.shape[0], cp, rv, nz, 1)
    H = restate(method, A0)
    if fam in ("random1", "random2", "random9", "random10"):
        assert H.sizes() == [A.shape[0]]                 # n <= max_coarse: one level
    if fam == "star" and method == "sa":
        assert H.sizes() == [300, 1]                     # one aggregate
    if fam == "laplacian_components" and method == "sa":
        assert (H.levels[0]["agg"] < 0).any()            # singletons: empty rows of T
    if fam == "arrow" and method == "sa":
        assert H.sizes() == [2000, 543, 150, 41, 12, 4] and H.nnz()[1] == 543 * 543
    check_against_restatement(amg, ctx, method, H, A0)


# ---------------------------------------------------------------------------------------------------------------- (b)
@pytest.mark.parametrize("fam,method", EXACT, ids=["%s-%s" % c for c in EXACT])
def test_setup_arithmetic_bit_for_bit(nls, ctx, fam, method):
    """From the device's exported A_l, P_l and T_l: A P and R (A P) as fma folds in the documented order, SA's T, rho, A T and
    P, RS's interpolation weights, each in the device's operations; every value must match bit for bit."""
    A = family(fam)
    amg, cp, rv, nz = make(nls, ctx, method, A)
    assert amg.setup(ctx.to_device(nz)) == 0
    ns, As, Ps, Ts = export(amg)
    H = restate(method, am.csr_of_csc(A.shape[0], cp, rv, nz, 1))
    assert ns == H.sizes()
    b = [1.0] * ns[0]
    for l in range(len(ns) - 1):
        A, P = As[l], Ps[l]
        if method == "sa":
            T = Ts[l]
            agg = -np.ones(ns[l], dtype=np.int64)
            agg[ax.rows_of(T)] = T.indices
            tval, nrm = ax.tentative_exact(agg, b)
            assert same_bits([T.data], [tval]), "T_%d" % l
            b = nrm.tolist()
            AT = ax.at_exact(A, T)
            assert same_pattern(AT, P), l                 # pattern(P) = pattern(A T)
            assert same_bits([P.data], [ax.sa_p_exact(A, T, AT, 4.0 / 3.0)]), "P_%d" % l
        else:
            assert same_bits([P.data], [ax.rs_p_exact(A, P, H.levels[l]["cf"])]), "P_%d" % l
        _, Ac = ax.galerkin_exact(A, P)
        assert same_pattern(Ac, As[l + 1]), l + 1
        assert same_bits([As[l + 1].data], [Ac.data]), "A_%d" % (l + 1)


# ---------------------------------------------------------------------------------------------------------------- (c)
def _random_values(A, seed):
    """Independent values on A's pattern (CSR order): standard normal off the diagonal, 4 + U(0, 1) on it."""
    rng = np.random.default_rng(seed)
    B = A.copy()
    B.data = rng.standard_normal(A.nnz)
    d = B.indices == ax.rows_of(B)
    B.data[d] = 4.0 + rng.random(int(d.sum()))
    return B


@pytest.mark.parametrize("fam,method", CASES, ids=IDS)
def test_refresh_at_random_values_within_the_componentwise_bound(nls, ctx, fam, method):
    """A refresh on the frozen pattern at independent random values (every pair-list term visible): every P_l and A_{l+1}
    within the componentwise bounds computed from the device's own A_l, P_l, T_l."""
    A = family(fam)
    amg, cp, rv, nz = make(nls, ctx, method, A)
    assert amg.setup(ctx.to_device(nz)) == 0
    H = restate(method, am.csr_of_csc(A.shape[0], cp, rv, nz, 1))
    B = _random_values(A, 99)
    _, _, nzb = _csc_of(B)
    assert amg.setup(ctx.to_device(nzb), rebuild=False) == 0
    ns, As, Ps, Ts = export(amg)
    assert ns == H.sizes() and same_bits([As[0].data], [am.csr_of_csc(A.shape[0], cp, rv, nzb, 1).data])
    check_values(method, ns, As, Ps, Ts, [L.get("cf") for L in H.levels])


# ---------------------------------------------------------------------------------------------------------------- (d)
@pytest.mark.parametrize("fam,method", FORMS, ids=["%s-%s" % c for c in FORMS])
def test_power_of_two_scaling_is_exact(nls, ctx, fam, method):
    """A -> 2^k A, k = +-20: every step scales exactly or is scale-invariant, so T, the aggregates or splitting and P are
    bit-identical, every A_l is exactly 2^k times the original, and one cycle exactly 2^-k times."""
    A = family(fam)
    amg, cp, rv, nz = make(nls, ctx, method, A)
    assert amg.setup(ctx.to_device(nz)) == 0
    ns, As, Ps, Ts = export(amg)
    b = ctx.to_device(np.random.default_rng(5).standard_normal(A.shape[0]))
    x = amg.solve(b).to_host()
    for k in (20, -20):
        s, _, _, _ = make(nls, ctx, method, A)
        assert s.setup(ctx.to_device(np.ldexp(nz, k))) == 0
        ns2, As2, Ps2, Ts2 = export(s)
        assert ns2 == ns
        assert same_bits(raw_of(Ps2 + Ts2), raw_of(Ps + Ts))
        assert same_bits(raw_of(As2), raw_of([sp.csr_matrix((np.ldexp(M.data, k), M.indices, M.indptr), shape=M.shape) for M in As]))
        assert same_bits([s.solve(b).to_host()], [np.ldexp(x, -k)])


def raw_of(Ms):
    return [a for M in Ms for a in (M.indptr, M.indices, M.data)]


# ---------------------------------------------------------------------------------------------------------------- (e)
@pytest.mark.parametrize("fam,method", FORMS, ids=["%s-%s" % c for c in FORMS])
def test_input_form_invariance(nls, ctx, fam, method):
    """Index base 0 or 1 and row indices shuffled within each CSC column give the same hierarchy and cycle, bit for bit."""
    A = family(fam)
    n = A.shape[0]
    b = ctx.to_device(np.random.default_rng(6).standard_normal(n))
    amg, cp, rv, nz = make(nls, ctx, method, A, base=1)
    assert amg.setup(ctx.to_device(nz)) == 0
    ref, xref = raw(amg), amg.solve(b).to_host()
    z, cp0, rv0, nz0 = make(nls, ctx, method, A, base=0)
    assert z.setup(ctx.to_device(nz0)) == 0
    assert same_bits(raw(z), ref) and same_bits([z.solve(b).to_host()], [xref])
    rng = np.random.default_rng(7)
    perm = np.concatenate([cp[j] - 1 + rng.permutation(cp[j + 1] - cp[j]) for j in range(n)]).astype(np.int64)
    cls = nls.SparseAMG.smoothed_aggregation if method == "sa" else nls.SparseAMG
    sh = cls(ctx, n, cp, rv[perm], 1)
    assert sh.setup(ctx.to_device(nz[perm])) == 0
    assert same_bits(raw(sh), ref) and same_bits([sh.solve(b).to_host()], [xref])


# ---------------------------------------------------------------------------------------------------------------- (f)
def _export_refused(nls, ctx, amg, what):
    L = nls.abi.lib()
    rowptr = np.zeros(amg.n + 1, dtype=np.int32)
    return L.b200_amg_export(amg._h, 0, what, rowptr.ctypes.data_as(C.c_void_p), None, None) == nls.abi.ERR_INVALID


@pytest.mark.parametrize("n", [1, 2, 9, 10])
@pytest.mark.parametrize("method", METHODS)
def test_single_level(nls, ctx, method, n):
    """n <= max_coarse: one level, no P or T to export, and the cycle is the coarsest inverse.  Its result against
    numpy.linalg.solve: the explicit inverse from LU is within gamma(3n) |A^-1| |L| |U| |X| of A^-1 and its GEMV adds
    gamma(n) |X| |b| (amg_exact.Cycle); LAPACK's solve is within gamma(3n) |A^-1| |L| |U| |x| of the solution."""
    A = family("random%d" % n)
    amg, cp, rv, nz = make(nls, ctx, method, A)
    assert amg.setup(ctx.to_device(nz)) == 0
    assert amg.levels()[0] == [n]
    assert _export_refused(nls, ctx, amg, nls.abi.AMG_EXPORT_P) and _export_refused(nls, ctx, amg, nls.abi.AMG_EXPORT_T)
    b = np.random.default_rng(n).standard_normal(n)
    x = amg.solve(ctx.to_device(b)).to_host()
    D = A.toarray()
    xs = np.linalg.solve(D, b)
    cyc = ax.Cycle([], [], A, 2.0 / 3.0, 1, 1)
    _, e = cyc._apply(b, np.zeros(n), 0)
    Pm, L, Uf = sla.lu(D)
    e_solve = ax.gamma(3 * n) * (np.abs(cyc.X) @ (np.abs(L) @ np.abs(Uf)) @ np.abs(xs))
    # e bounds the device's result and e_solve LAPACK's, each against the exact solution, so their sum (not twice either)
    # bounds the difference; both are first order, and 1.1 covers the second-order remainder, a relative O(n u) << 0.1
    within(x, xs, 1.1 * (e + e_solve), "single-level solve")


@pytest.mark.parametrize("max_levels", [1, 2, 3])
@pytest.mark.parametrize("method", METHODS)
def test_max_levels(nls, ctx, method, max_levels):
    A = random_matrix(1500, 21)
    amg, cp, rv, nz = make(nls, ctx, method, A, max_levels=max_levels)
    assert amg.setup(ctx.to_device(nz)) == 0
    A0 = am.csr_of_csc(1500, cp, rv, nz, 1)
    H = restate(method, A0, max_levels=max_levels)
    assert len(H.sizes()) == max_levels
    check_against_restatement(amg, ctx, method, H, A0)


@pytest.mark.parametrize("method", METHODS)
def test_a_level_landing_exactly_on_max_coarse(nls, ctx, method):
    """max_coarse equal to level 1's size stops there; one less goes on coarsening."""
    A = random_matrix(1500, 22)
    A0 = am.csr_of_csc(1500, *_csc_of(A))
    s1 = restate(method, A0).sizes()[1]
    for mc, nlev in ((s1, 2), (s1 - 1, None)):
        amg, cp, rv, nz = make(nls, ctx, method, A, max_coarse=mc)
        assert amg.setup(ctx.to_device(nz)) == 0
        H = restate(method, A0, max_coarse=mc)
        assert (len(H.sizes()) == nlev) if nlev else (len(H.sizes()) > 2)
        check_against_restatement(amg, ctx, method, H, A0)


OPTIONS = [dict(theta=0.0), dict(theta=1.0), dict(presweeps=0, postsweeps=0), dict(presweeps=0, postsweeps=3),
           dict(presweeps=3, postsweeps=0), dict(presweeps=3, postsweeps=3), dict(omega=0.5), dict(omega=1.0)]
SA_OPTIONS = [dict(smooth_omega=0.5), dict(smooth_omega=4.0 / 3.0, theta=0.25)]


@pytest.mark.parametrize("method,opts", [(m, o) for m in METHODS for o in OPTIONS] + [("sa", o) for o in SA_OPTIONS],
                         ids=lambda v: v if isinstance(v, str) else "-".join("%s=%g" % kv for kv in v.items()))
def test_options_against_the_restatement(nls, ctx, method, opts):
    A = ax.with_stored_zeros(random_matrix(1200, 23), 23)
    amg, cp, rv, nz = make(nls, ctx, method, A, **opts)
    assert amg.setup(ctx.to_device(nz)) == 0
    A0 = am.csr_of_csc(1200, cp, rv, nz, 1)
    # Ruge-Stueben at theta = 0 makes every nonzero strong, so on a coarse level the splitting turns on which Galerkin values
    # are exactly 0.0; the restatement's scipy sums round differently from the device's fma folds (which test (b) restates bit
    # for bit), and from level 2 on the two hierarchies differ by that alone.  The rules are then checked level by level on the
    # device's own A_l.
    stepwise = method == "rs" and opts.get("theta") == 0.0
    check_against_restatement(amg, ctx, method, restate(method, A0, **opts), A0, opts=opts, stepwise=stepwise)
    if not stepwise:
        ns, As, Ps, Ts = export(amg)
        check_steps(method, ns, As, Ps, Ts, opts)


# ---------------------------------------------------------------------------------------------------------------- (g)
def _with(A, entries):
    B = A.tolil(copy=True)
    for (i, j), v in entries.items():
        B[i, j] = v
    return ax._sorted(B)


@pytest.mark.parametrize("method", METHODS)
def test_info_codes(nls, ctx, method):
    """info (DESIGN.md §4h): the 1-based level of a zero or non-finite diagonal or lumped denominator, or the coarsest level at
    an exactly zero LU pivot; the next setup at good values returns 0 and matches the restatement."""
    A = random_matrix(300, 31)
    assert len(restate(method, A).sizes()) >= 2
    cp, rv, nz = _csc_of(A)
    amg, _, _, _ = make(nls, ctx, method, A)
    d = np.flatnonzero(rv - 1 == np.repeat(np.arange(300), np.diff(cp)))
    for v in (0.0, np.nan, np.inf, -np.inf):
        bad = nz.copy()
        bad[d[17]] = v
        assert amg.setup(ctx.to_device(bad)) == 1, v
        assert amg.setup(ctx.to_device(nz)) == 0
        check_against_restatement(amg, ctx, method, restate(method, A), A)
    # a single level with an exactly zero LU pivot: the block [[1, 1], [1, 1]]
    S = _with(sp.identity(6, format="lil") * 3.0, {(0, 0): 1.0, (0, 1): 1.0, (1, 0): 1.0, (1, 1): 1.0})
    one, cp1, rv1, nz1 = make(nls, ctx, method, S)
    assert one.setup(ctx.to_device(nz1)) == 1 and one.levels()[0] == [6]
    good = _with(S, {(1, 1): 2.0})
    _, _, nzg = _csc_of(good)
    assert one.setup(ctx.to_device(nzg)) == 0
    check_against_restatement(one, ctx, method, restate(method, good), good)


@pytest.mark.parametrize("method", METHODS)
def test_single_level_non_finite_diagonal(nls, ctx, method):
    """On a single level 1/diag is never formed, so only the LU can notice a non-finite diagonal.  Pinned: a NaN pivot makes
    getrf report it (info 1); an infinite one is a nonzero pivot, so setup reports 0 and the inverse it builds is finite
    (x_2 = (y_2 - ...) / inf = 0): a caller is not told that the matrix held an infinity."""
    S = sp.identity(6, format="lil") * 3.0
    S[2, 3] = S[3, 2] = -1.0
    for v, info in ((np.nan, 1), (np.inf, 0), (-np.inf, 0)):
        B = _with(S, {(2, 2): v})
        amg, cp, rv, nz = make(nls, ctx, method, B)
        assert amg.setup(ctx.to_device(nz)) == info and amg.levels()[0] == [6], v
        if info == 0:
            x = amg.solve(ctx.to_device(np.ones(6))).to_host()
            assert np.isfinite(x).all() and x[2] == 0.0, v


def test_rs_zero_lumped_denominator(nls, ctx):
    """An F row with a_ii = -0.1, one weak positive off-diagonal 0.1 and strong negative C neighbours: no positive entry among
    its interpolatory set, so 0.1 is lumped into a_ii = -0.1, the denominator is exactly 0 and info names level 1 (a_ii itself
    is not zero).  The same pattern at good values (the extra entry a stored 0.0) then sets up with info 0."""
    n = 40
    chain = sp.diags([-np.ones(n - 1), 2.0 * np.ones(n), -np.ones(n - 1)], [-1, 0, 1], shape=(n, n)).tocoo()
    cf = am.split(ax._sorted(chain), am.strength(ax._sorted(chain)))
    i = next(i for i in range(15, 25) if not cf[i] and cf[i - 1] and cf[i + 1])
    k = i + 10

    def with_values(aii, aik):
        v = np.where(chain.row == chain.col, np.where(chain.row == i, aii, chain.data), chain.data)
        return ax._sorted(sp.coo_matrix((np.r_[v, aik], (np.r_[chain.row, i], np.r_[chain.col, k])), shape=(n, n)))

    good, bad = with_values(2.0, 0.0), with_values(-0.1, 0.1)
    assert good.nnz == bad.nnz == chain.nnz + 1
    assert np.array_equal(am.split(bad, am.strength(bad)), cf)           # the same splitting: 0.1 is weak
    amg, cp, rv, nz = make(nls, ctx, "rs", bad)
    assert amg.setup(ctx.to_device(nz)) == 1
    _, _, nzg = _csc_of(good)
    assert amg.setup(ctx.to_device(nzg)) == 0
    check_against_restatement(amg, ctx, "rs", am.Hierarchy(good), good)


# ---------------------------------------------------------------------------------------------------------------- (h)
@pytest.mark.parametrize("method", METHODS)
def test_rebuild_at_new_level_sizes_replays_a_new_graph(nls, ctx, method):
    """Rebuild, solve (captures the cycle graph), rebuild at values whose hierarchy has other level sizes, solve: the second
    cycle must be that of the new hierarchy (a graph kept from the first would read freed, possibly reused buffers)."""
    A = random_matrix(1000, 41)
    B = _random_values(A, 42)
    B.data *= np.where(B.indices == ax.rows_of(B), 0.25, 1.0)
    HA, HB = restate(method, A), restate(method, B)
    assert HA.sizes() != HB.sizes()
    amg, cp, rv, nz = make(nls, ctx, method, A)
    assert amg.setup(ctx.to_device(nz)) == 0
    check_against_restatement(amg, ctx, method, HA, A, seed=3)
    _, _, nzb = _csc_of(B)
    assert amg.setup(ctx.to_device(nzb)) == 0
    check_against_restatement(amg, ctx, method, HB, B, seed=3)
    assert amg.setup(ctx.to_device(nz)) == 0
    check_against_restatement(amg, ctx, method, HA, A, seed=4)


@pytest.mark.parametrize("method", METHODS)
def test_refresh_at_values_that_would_change_the_strength_graph(nls, ctx, method):
    """A refresh keeps the splitting / aggregates even where the new values would choose others: it equals the restatement's
    frozen refresh."""
    A = random_matrix(1000, 43)
    B = _random_values(A, 44)
    H = restate(method, A)
    assert restate(method, B).sizes() != H.sizes()
    amg, cp, rv, nz = make(nls, ctx, method, A)
    assert amg.setup(ctx.to_device(nz)) == 0
    _, _, nzb = _csc_of(B)
    assert amg.setup(ctx.to_device(nzb), rebuild=False) == 0
    check_against_restatement(amg, ctx, method, H.refresh(B), B)


@pytest.mark.parametrize("method", METHODS)
def test_direct_launches_equal_the_graph_replay(nls, ctx, method):
    """A handle whose first solve runs under profiling launches the cycle directly (no graph is captured); its results are
    the bits of a handle that replays the captured graph."""
    A = family("laplacian_components")
    b = ctx.to_device(np.random.default_rng(8).standard_normal(A.shape[0]))
    g, cp, rv, nz = make(nls, ctx, method, A)
    assert g.setup(ctx.to_device(nz)) == 0
    xg = [g.solve(b).to_host() for _ in range(2)]
    d, _, _, _ = make(nls, ctx, method, A)
    assert d.setup(ctx.to_device(nz)) == 0
    ctx.profile(True)
    try:
        xd = [d.solve(b).to_host() for _ in range(2)]
    finally:
        ctx.profile(False)
    assert same_bits(xg, xd) and same_bits(xg[:1], xg[1:])


# ---------------------------------------------------------------------------------------------------------------- (i)
@pytest.mark.parametrize("side", ["left", "right"])
@pytest.mark.parametrize("method", METHODS)
def test_preconditioned_gmres_matches_the_oracle(nls, ctx, po, method, side):
    """GMRES on a non-symmetric n = 1500 CSC matrix with the AMG cycle as Pl or Pr, against the oracle's GMRES on the dense
    M^-1 A (left) or A M^-1 (right), M^-1 the cycle of the device's own hierarchy applied to the identity.

    Tolerances: the iteration counts within 1; rnorm0 (|| M^-1 b || left, || b || right) within the norm of the cycle bound
    plus gamma(n) of itself; left, the solutions within 2.2 ||K^-1|| (rtol r0 + n u ||K|| ||x||), K the
    preconditioned operator: each side's residual is below rtol r0 up to GMRES's backward error n u ||K|| ||y||; right
    preconditioning solves A x = b to rtol ||b|| plus that and the error ||A|| ||e_y|| of the final x = M^-1 y, so there the
    bound is 2.2 ||A^-1|| (rtol ||b|| + n u ||K|| ||y|| + ||A|| ||e_y||)."""
    n = 1500
    A = random_matrix(n, 51)
    amg, cp, rv, nz = make(nls, ctx, method, A)
    assert amg.setup(ctx.to_device(nz)) == 0
    ns, As, Ps, Ts = export(amg)
    assert len(ns) >= 2
    cyc = ax.Cycle(As[:-1], Ps, As[-1])
    Minv = cyc(np.eye(n))
    D = A.toarray()
    b = np.random.default_rng(52).standard_normal(n)
    rtol = 1e-10
    opts = po.default_gmres_opts(atol=0.0, rtol=rtol, orth=po.ORTH_CGS2)
    gm = nls.GmresSolver(ctx, n, nls.KrylovJL_GMRES(orth="cgs2"), atol=0.0, rtol=rtol)
    csc = ("csc", ctx.to_device(cp, np.int64), ctx.to_device(rv, np.int64), ctx.to_device(nz), 1)
    if side == "left":
        K = Minv @ D
        rhs, eb = cyc.bound(b)
        xo, so = po.gmres(rhs, dense=K, opts=opts)
        x, st = gm.solve(csc, ctx.to_device(b), Pl=amg.linop())
        r0_bound = np.linalg.norm(eb) + ax.gamma(n) * so.rnorm0
        sv = np.linalg.svd(K, compute_uv=False)
        err = 2.2 / sv[-1] * (rtol * so.rnorm0 + n * ax.U * sv[0] * np.linalg.norm(xo))
        xref = xo
    else:
        K = D @ Minv
        xo, so = po.gmres(b, dense=K, opts=opts)
        x, st = gm.solve(csc, ctx.to_device(b), Pr=amg.linop())
        r0_bound = 2 * ax.gamma(n) * so.rnorm0
        xref, ey = cyc.bound(xo)                  # x = M^-1 y, one more cycle
        sk, sd = np.linalg.svd(K, compute_uv=False), np.linalg.svd(D, compute_uv=False)
        err = 2.2 / sd[-1] * (rtol * so.rnorm0 + n * ax.U * sk[0] * np.linalg.norm(xo) + sd[0] * np.linalg.norm(ey))
    assert st.status == nls.abi.LS_SOLVED == so.status and abs(st.iters - so.iters) <= 1
    assert abs(st.rnorm0 - so.rnorm0) <= r0_bound
    assert np.linalg.norm(x.to_host() - xref) <= err


# ---------------------------------------------------------------------------------------------------------------- (j)
def test_product_term_guard(nls, ctx):
    """The weak-hub arrow at n = 100 000: level 0's A P has 2 750 319 962 terms (tests/test_amg_exact.py), past the int32
    guard, which runs on the int64 count before anything is allocated by it.  Setup fails cleanly, the handle refuses what
    needs a hierarchy, and the context still builds and solves another handle."""
    A = ax.arrow(100_000)
    amg, cp, rv, nz = make(nls, ctx, "sa", A)
    with pytest.raises(nls.abi.B200Error) as e:
        amg.setup(ctx.to_device(nz))
    assert e.value.code == nls.abi.ERR_UNSUPPORTED and "2^31 or more" in str(e.value)
    for call in (amg.levels, lambda: amg.level(0), lambda: amg.solve(ctx.to_device(np.ones(A.shape[0])))):
        with pytest.raises(nls.abi.B200Error) as e:
            call()
        assert e.value.code == nls.abi.ERR_INVALID
    B = family("random257")
    other, cp, rv, nz = make(nls, ctx, "sa", B)
    assert other.setup(ctx.to_device(nz)) == 0
    check_against_restatement(other, ctx, "sa", sa.Hierarchy(B), B)


# ---------------------------------------------------------------------------------------------------------------- stop advice
@pytest.mark.parametrize("method", METHODS)
def test_a_stalled_coarsening_says_so(nls, ctx, method):
    """Above the dense cap, the advice names the cause: a level with no strong connection stalls (raising max_levels cannot
    help), max_coarse above the cap asks to lower it, and a max_levels stop keeps its advice."""
    n = 5000
    rng = np.random.default_rng(61)
    D = ax._sorted(sp.diags(1.0 + rng.random(n)))          # no off-diagonal: no strong connection anywhere
    amg, cp, rv, nz = make(nls, ctx, method, D)
    with pytest.raises(nls.abi.B200Error) as e:
        amg.setup(ctx.to_device(nz))
    msg = str(e.value)
    assert e.value.code == nls.abi.ERR_UNSUPPORTED and "stalls at level 1" in msg and "5000" in msg and "max_levels" not in msg
    assert ("no aggregate" if method == "sa" else "no C point") in msg
    A = random_matrix(n, 62)
    amg, cp, rv, nz = make(nls, ctx, method, A, max_coarse=6000)
    with pytest.raises(nls.abi.B200Error) as e:
        amg.setup(ctx.to_device(nz))
    assert e.value.code == nls.abi.ERR_UNSUPPORTED and "lower max_coarse" in str(e.value) and "max_levels" not in str(e.value)
    amg, cp, rv, nz = make(nls, ctx, method, A, max_levels=1)
    with pytest.raises(nls.abi.B200Error) as e:
        amg.setup(ctx.to_device(nz))
    assert e.value.code == nls.abi.ERR_UNSUPPORTED and "raise max_levels" in str(e.value)
    amg, cp, rv, nz = make(nls, ctx, method, A)          # the same handle type coarsens a coupled matrix of that size
    assert amg.setup(ctx.to_device(nz)) == 0
