"""The exact restatements and bounds of oracle/amg_exact.py, pinned on the CPU: the fma emulator is fused (one rounding), the
exact restatements of each setup step agree with the NumPy restatements within the derived bounds, the cycle bound holds, and
the matrix families of tests/test_gpu_amg_general.py have the shapes those tests rely on."""
from fractions import Fraction

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import amg_exact as ax
from oracle import amg_numpy as am
from oracle import sa_numpy as sa
from test_amg_oracle import random_matrix


def test_fma_rounds_once():
    a, b = 1.0 + 2.0 ** -30, 1.0 - 2.0 ** -30      # a b = 1 - 2^-60: rounds to 1.0 as a product
    assert a * b - 1.0 == 0.0
    assert ax.fma(a, b, -1.0) == -(2.0 ** -60)
    # double rounding: a b = 1 + 2^-53 - 2^-105 rounds down to 1, but a b + 2^-104 lies above the tie and rounds up
    a, b, s = 1.0 + 2.0 ** -52, 1.0 - 2.0 ** -53, 2.0 ** -104
    assert ax.fma(a, b, s) == 1.0 + 2.0 ** -52 and a * b + s == 1.0
    assert ax.fma(a, b, s) != a * b + s and ax.fma(a, b, s) == float(Fraction(a) * Fraction(b) + Fraction(s))
    assert str(ax.fma(0.0, -1.0, -0.0)) == "-0.0" and str(ax.fma(1.0, 1.0, -1.0)) == "0.0"


def test_fma_equals_the_rational_rounding():
    rng = np.random.default_rng(0)
    for a, b, s in (rng.standard_normal(3) * np.ldexp(1.0, rng.integers(-40, 40, 3)) for _ in range(2000)):
        a, b, s = float(a), float(b), float(s)
        assert ax.fma(a, b, s) == float(Fraction(a) * Fraction(b) + Fraction(s))


SMALL = {"random257": lambda: random_matrix(257, 268), "one_sided": lambda: ax.one_sided(300, 1),
         "laplacian_components": lambda: ax.laplacian_components(600, 2), "star": lambda: ax.star(300, 3),
         "stored_zeros": lambda: ax.with_stored_zeros(random_matrix(800, 4), 4),
         "rows_scaled": lambda: ax.rows_scaled(random_matrix(800, 5), 5)}


@pytest.mark.parametrize("method", ["rs", "sa"])
@pytest.mark.parametrize("fam", sorted(SMALL))
def test_exact_steps_within_the_bounds_of_the_restatement(fam, method):
    """On the restatement's own hierarchy: the exact restatement of every step (the device's operations, one rounding each)
    has the restated patterns and lies within the derived bound of the restated values, and SA's T is the restated T bit for
    bit; the cycle bound holds between two evaluations."""
    A = SMALL[fam]()
    H = (sa.Hierarchy if method == "sa" else am.Hierarchy)(A)
    assert len(H.levels) >= 1
    b = [1.0] * A.shape[0]
    for l, L in enumerate(H.levels):
        Al, P = L["A"], L["P"]
        Ac = H.levels[l + 1]["A"] if l + 1 < len(H.levels) else H.coarse
        if method == "sa":
            T = L["T"]
            tval, nrm = ax.tentative_exact(L["agg"], b)
            assert np.array_equal(tval, T.data)
            b = nrm.tolist()
            AT = ax.at_exact(Al, T)
            assert np.array_equal(AT.indptr, P.indptr) and np.array_equal(AT.indices, P.indices)
            ref, bnd = ax.sa_p_bound(Al, T, P, 4.0 / 3.0)
            got = ax.sa_p_exact(Al, T, AT, 4.0 / 3.0)
        else:
            ref, bnd = ax.rs_p_bound(Al, P, L["cf"])
            got = ax.rs_p_exact(Al, P, L["cf"])
        assert np.all(np.abs(got - P.data) <= bnd) and np.all(np.abs(ref - P.data) <= bnd)
        _, Ace = ax.galerkin_exact(Al, P)
        assert np.array_equal(Ace.indptr, Ac.indptr) and np.array_equal(Ace.indices, Ac.indices)
        ref, bnd = ax.galerkin_bound(Al, P, Ac)
        assert np.all(np.abs(Ace.data - ref) <= bnd) and np.all(np.abs(Ac.data - ref) <= bnd)
    cyc = ax.Cycle([L["A"] for L in H.levels], [L["P"] for L in H.levels], H.coarse)
    x = np.random.default_rng(1).standard_normal(A.shape[0])
    y, bnd = cyc.bound(x)
    assert np.all(np.abs(y - H.cycle(x)) <= bnd)


def test_a_bound_sees_a_missing_term():
    """Dropping one term of one Galerkin entry moves it outside the bound (the bound is not loose at that scale)."""
    A = random_matrix(257, 268)
    H = am.Hierarchy(A)
    L = H.levels[0]
    Ac = H.levels[1]["A"]
    ref, bnd = ax.galerkin_bound(L["A"], L["P"], Ac)
    P = L["P"].tolil()
    r, c = next((r, c) for r, c in zip(*L["P"].nonzero()) if not L["cf"][r])
    P[r, c] = 0.0
    _, bad = ax.galerkin_exact(L["A"], sp.csr_matrix(P))
    moved = np.abs(ax.on_pattern(Ac, bad) - ref) > bnd
    assert moved.any()


def test_the_families():
    A = ax.one_sided(300, 1)
    assert np.array_equal(np.unique(A.indices - ax.rows_of(A)), [0, 1])
    S = ax.with_stored_zeros(random_matrix(800, 4), 4)
    off = S.indices != ax.rows_of(S)
    assert (S.data[off] == 0.0).sum() == int(0.05 * off.sum())
    R = ax.rows_scaled(random_matrix(800, 5), 5)
    e = np.frexp(R.data / random_matrix(800, 5).data)
    assert np.all(e[0] == 0.5)                                    # rows scaled by powers of two, exactly
    L = ax.laplacian_components(600, 2)
    assert np.abs(np.asarray((L - 0.1 * sp.identity(600)).sum(axis=1))).max() <= 1e-12 * abs(L).max()
    assert (np.diff(L.indptr) == 1).sum() >= 5                    # singletons
    G = sa.strength_graph(ax.star(300, 3))
    assert np.diff(G.indptr)[0] == 299                            # every hub entry strong
    assert sa.Hierarchy(ax.star(300, 3)).sizes() == [300, 1]
    for n in (65536, 65537):                                      # the key-width members: banded, no coarse fill
        B = ax.banded(n, n)
        assert (n * n - 1).bit_length() == (32 if n == 65536 else 33)
        for H in (am.Hierarchy(B), sa.Hierarchy(B)):
            assert H.sizes()[-1] <= 4096 and max(H.nnz()) == B.nnz


def test_arrow_hierarchy():
    """The weak-hub arrow at n = 2000 (DESIGN.md §4i rules): the hub is isolated, so T's row 0 is empty while A T's row 0 is
    dense; level 1 fills in completely and its A P has 44 M terms."""
    A = ax.arrow(2000)
    H = sa.Hierarchy(A)
    assert H.sizes() == [2000, 543, 150, 41, 12, 4]
    assert H.nnz()[1] == 543 * 543
    T, P = H.levels[0]["T"], H.levels[0]["P"]
    assert T.indptr[1] == 0 and np.diff(P.indptr)[0] == 543
    L1 = H.levels[1]
    terms = int((ax.ones(L1["A"]) @ np.diff(L1["P"].indptr)).sum())
    assert terms == 44_227_350


def test_arrow_at_100k_passes_the_product_guard():
    """At n = 100 000 level 0's A P has 2^31 or more terms: the restatement's aggregates give P a dense row 0, and every row
    of A holds column 0."""
    A = ax.arrow(100_000)
    G = sa.strength_graph(A)
    agg, na, _, _ = sa.aggregate(G)
    assert na == 27_497 and agg[0] == -1
    T, _ = sa.tentative(agg, na, np.ones(A.shape[0]))
    Pn = np.diff((ax.ones(A) @ ax.ones(T)).indptr)
    terms = int((ax.ones(A) @ Pn).sum())
    assert terms == 2_750_319_962 and terms >= 2 ** 31


@pytest.mark.parametrize("seed", range(8))
def test_a_level_with_a_strong_connection_always_reduces(seed):
    """The no-reduction stall (every point a C point, every node an aggregate root) needs no strong connection at all: the
    first C point's dependents become F, and a root's neighbours are never roots.  Pinned on both restatements."""
    n = [5, 12, 40, 100, 300, 600, 1000, 2000][seed]
    for A in (random_matrix(n, seed), ax.one_sided(n, seed), ax.banded(n, seed)):
        strong = am.strength(A)
        if strong.any():
            assert 0 < am.split(A, strong).sum() < n
        G = sa.strength_graph(A)
        if G.nnz:
            _, na, _, _ = sa.aggregate(G)
            assert 0 < na < n
