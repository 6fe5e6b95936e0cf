"""CPU tests of the Brusselator stencil launch plan (csrc/problems.cu, stencil_plan and bruss3d_ring_kernel's producer prologue),
restated here so that tests/test_gpu_stencil.py can pick one grid size per launch regime and check that the library plans
exactly what this restatement does.

A 3D op with a ring instantiation (residual, residual + norm, JVP, VJP) runs the halo-ring kernel when N is even,
N^2 >= TS_L + 2N, the ring holds R >= 4 plane slots, and no CTA's run of plane-chunks is longer than 3N; otherwise, and for
every 2D op, the thread-per-cell kernel.  The chunks * N plane-chunks are dealt out in contiguous runs to a one-wave grid of
min(2 SMs, W / 2) CTAs, and a CTA marches once per chunk its run touches."""
import numpy as np
import pytest

TS_L = 512          # flat plane positions per chunk (two per consumer thread)
TS_MAXR = 8
TS_MAXMARCH = 4
PB_THREADS = 256
RING_BYTES = 100 * 1024
OPS = ("residual", "residual_norm", "jvp", "vjp")   # index == B200_STENCIL_*
SM_COUNTS = (132, 114)                              # H100 SXM, H100 PCIe


def cdiv(a, b):
    return -(-a // b)


def exact_alpha(N, k):
    """alpha such that the library's a = alpha / (dx * dx) is exactly 2**k (dx = 1 / (N - 1) as in create_bruss)."""
    dx = 1.0 / (N - 1)
    return 2.0 ** k * (dx * dx)


def ring_geometry(N, op):
    """(ring slots R, chunks, W = chunks * N) of the 3D ring kernel, before any fallback test."""
    has_y = OPS[op] in ("jvp", "vjp")
    slot = 8 * (2 * (TS_L + 2 * N) + (2 * TS_L if has_y else 0))
    chunks = cdiv(N * N, TS_L)
    return min(TS_MAXR, RING_BYTES // slot), chunks, chunks * N


def fallback_cause(dim, N, op, sm_count):
    """Why an op runs the plain kernel ("2d", "odd", "small", "depth", "run"), or None for the ring kernel."""
    if dim == 2:
        return "2d"
    if N * N < TS_L + 2 * N:
        return "small"
    if N % 2:
        return "odd"
    R, _, W = ring_geometry(N, op)
    if R < 4:
        return "depth"
    grid = max(1, min(2 * sm_count, W // 2))
    if cdiv(W, grid) > (TS_MAXMARCH - 1) * N:
        return "run"
    return None


def marches(N, W, grid, b):
    """The producer prologue of CTA b: [(chunk, ka, m, l0)], stopping (as the kernel does) after TS_MAXMARCH marches."""
    w0, w1 = W * b // grid, W * (b + 1) // grid
    out, l = [], 0
    while w0 < w1 and len(out) < TS_MAXMARCH:
        c, ka = divmod(w0, N)
        m = min(N - ka, w1 - w0)
        out.append((c, ka, m, l))
        l += m + 2
        w0 += m
    return out


def plan(dim, N, op, sm_count):
    """(ring_slots, grid, max_marches) exactly as b200_problem_stencil_plan reports it."""
    NC = N ** dim
    if fallback_cause(dim, N, op, sm_count) is not None:
        return 0, cdiv(NC, PB_THREADS), 0
    R, _, W = ring_geometry(N, op)
    grid = max(1, min(2 * sm_count, W // 2))
    return R, grid, max(len(marches(N, W, grid, b)) for b in range(grid))


def ring_layout(N, op, sm_count):
    """(grid, W, [marches of every CTA]) of a ring launch."""
    R, _, W = ring_geometry(N, op)
    grid = max(1, min(2 * sm_count, W // 2))
    return grid, W, [marches(N, W, grid, b) for b in range(grid)]


# ---- launch regimes.  A class is (family, feature, value); family "residual" covers residual and residual + norm (one plan),
#      "tangent" covers JVP and VJP.
FAMILY_OP = {"residual": 0, "tangent": 2}


def classify(N, family, sm_count):
    """The set of regime classes the 3D op family at N falls in."""
    op = FAMILY_OP[family]
    cause = fallback_cause(3, N, op, sm_count)
    if cause is not None:
        return {(family, "fallback", cause)}
    R, grid, mm = plan(3, N, op, sm_count)
    _, chunks, W = ring_geometry(N, op)
    out = {(family, "R", R), (family, "marches", mm), (family, "last_chunk", "exact" if (N * N) % TS_L == 0 else "ragged")}
    if grid == W // 2 and grid < 2 * sm_count:
        out.add((family, "grid", "W/2"))
    if TS_L < N:
        out.add((family, "chunk", "shorter_than_row"))
    return out


def required_classes(sm_count):
    """Every regime of the launch table a 132- or 114-SM H100 reaches (the run-length fallback is unreachable there)."""
    req = {("residual", "R", r) for r in (4, 5, 6, 7, 8)} | {("residual", "marches", m) for m in (1, 2, 3, 4)}
    req |= {("tangent", "R", r) for r in (4, 5)} | {("tangent", "marches", m) for m in (1, 2)}
    for fam in ("residual", "tangent"):
        req |= {(fam, "fallback", c) for c in ("odd", "small", "depth")}
        req |= {(fam, "last_chunk", "exact"), (fam, "last_chunk", "ragged"), (fam, "grid", "W/2")}
    req.add(("residual", "chunk", "shorter_than_row"))
    return req


EXTRA_N = (3, 4, 22, 32, 96, 128)   # the smallest sizes, the largest small fallback, and exact last chunks


def select_sizes(sm_count, nmax=1023):
    """{class: smallest 3D N in it} over every class reachable with N <= nmax, plus EXTRA_N under their own keys."""
    sel = {}
    for N in range(3, nmax + 1):
        for fam in FAMILY_OP:
            for c in classify(N, fam, sm_count):
                sel.setdefault(c, N)
    for N in EXTRA_N:
        sel[("extra", "N", N)] = N
    return sel


def family_sizes(sm_count, family):
    """Sorted distinct N the GPU tests run for one op family: the selected N of its classes and the extras."""
    sel = select_sizes(sm_count)
    return sorted({N for c, N in sel.items() if c[0] in (family, "extra")})


# ----------------------------------------------------------------------------- tests
@pytest.mark.parametrize("sm_count", SM_COUNTS)
def test_every_regime_exists_and_the_selector_hits_it(sm_count):
    sel = select_sizes(sm_count)
    missing = required_classes(sm_count) - set(sel)
    assert not missing, missing
    for c, N in sel.items():
        if c[0] != "extra":
            assert c in classify(N, c[0], sm_count), (c, N)
    for fam in FAMILY_OP:
        Ns = family_sizes(sm_count, fam)
        hit = set().union(*(classify(N, fam, sm_count) for N in Ns))
        assert {c for c in required_classes(sm_count) if c[0] == fam} <= hit
    # the run-length fallback never triggers before R < 4 on an H100
    assert not any(c[2] == "run" for c in sel if c[1] == "fallback")


@pytest.mark.parametrize("sm_count", SM_COUNTS)
def test_launch_table(sm_count):
    # the ring depth by N and the fallback boundaries do not depend on the SM count
    for N in range(24, 545, 2):
        R = plan(3, N, 0, sm_count)[0]
        assert R == (8 if N <= 144 else 7 if N <= 200 else 6 if N <= 276 else 5 if N <= 384 else 4), N
    for N in range(24, 289, 2):
        assert plan(3, N, 2, sm_count)[0] == (5 if N <= 128 else 4), N
    assert [N for N in range(3, 1025) if plan(3, N, 0, sm_count)[0]] == list(range(24, 545, 2))
    assert [N for N in range(3, 1025) if plan(3, N, 2, sm_count)[0]] == list(range(24, 289, 2))
    assert fallback_cause(3, 22, 0, sm_count) == "small" and fallback_cause(3, 546, 0, sm_count) == "depth"
    assert fallback_cause(3, 290, 2, sm_count) == "depth" and fallback_cause(3, 25, 0, sm_count) == "odd"
    for op in range(4):
        assert plan(3, 100, op, sm_count) == plan(3, 100, op ^ 1, sm_count)   # residual == residual + norm, JVP == VJP
        assert plan(2, 4097, op, sm_count) == (0, cdiv(4097 ** 2, PB_THREADS), 0)
    # W / 2 < 2 SMs exactly up to N = 64 (132 SMs) or 58 (114 SMs)
    assert max(N for N in range(24, 545, 2) if plan(3, N, 0, sm_count)[1] < 2 * sm_count) == {132: 64, 114: 58}[sm_count]


def test_launch_table_march_counts_h100():
    mm = {N: plan(3, N, 0, 132)[2] for N in range(24, 545, 2)}
    assert mm[64] == 1 and mm[66] == 2 and mm[72] == 1
    assert min(N for N in mm if mm[N] == 3) == 372 and min(N for N in mm if mm[N] == 4) == 522
    assert max(plan(3, N, 2, 132)[2] for N in range(24, 289, 2)) == 2


@pytest.mark.parametrize("sm_count", SM_COUNTS + (8, 1))
def test_marches_tile_every_run(sm_count):
    # every planned CTA covers its run exactly in at most TS_MAXMARCH marches, and the runs tile chunks * N with no gap: the
    # prologue stops silently at four marches, so a plan that needed a fifth would drop planes
    for op in (0, 2):
        for N in range(24, 1025, 2):
            if fallback_cause(3, N, op, sm_count) is not None:
                continue
            grid, W, ms = ring_layout(N, op, sm_count)
            w = 0
            for b, mlist in enumerate(ms):
                w0, w1 = W * b // grid, W * (b + 1) // grid
                assert w0 == w and w1 - w0 >= 2 and len(mlist) <= TS_MAXMARCH, (N, op, b)
                l = 0
                for c, ka, m, l0 in mlist:   # consecutive marches, each inside one chunk, continue where the last one ended
                    assert c * N + ka == w and 1 <= m <= N - ka and l0 == l, (N, op, b)
                    w += m
                    l += m + 2
                assert w == w1, (N, op, b)
            assert w == W, (N, op)


def test_run_length_fallback_on_a_small_gpu():
    # unreachable on an H100 (R < 4 comes first), so pinned on a hypothetical 8-SM part: the grid stays at 16 CTAs and a run
    # outgrows three chunk-lengths of planes from N = 158 on
    runs = [N for N in range(24, 545, 2) if fallback_cause(3, N, 0, 8) == "run"]
    assert runs == list(range(158, 545, 2))
    assert plan(3, 156, 0, 8)[0] == 7 and plan(3, 158, 0, 8) == (0, cdiv(158 ** 3, PB_THREADS), 0)
    for N in (runs[0], runs[0] + 20):
        grid, W, _ = ring_layout(N, 0, 8)
        assert cdiv(W, grid) > 3 * N


def test_exact_alpha_gives_a_power_of_two():
    for N in range(3, 1025):
        dx = 1.0 / float(N - 1)
        for k in (0, 3, 10):
            assert exact_alpha(N, k) / (dx * dx) == 2.0 ** k
    # the default alpha is not exact: a probe built on it would not be an integer computation
    assert 10.0 / ((1.0 / 23) * (1.0 / 23)) != 5290.0 and 10.0 / ((1.0 / 99) * (1.0 / 99)) != 98010.0


def forcing_plane(N):
    """brusselator_f on the (i, j) plane as create_bruss evaluates it: 5 inside the disk around (0.3, 0.6) of radius 0.1."""
    x = np.arange(N) / float(N - 1)
    dx2 = (x - 0.3) * (x - 0.3)
    dy2 = (x - 0.6) * (x - 0.6)
    return np.where(dx2[None, :] + dy2[:, None] <= 0.1 * 0.1, 5.0, 0.0)   # [j, i]


def test_forcing_plane():
    f = forcing_plane(24)
    assert f.shape == (24, 24) and set(np.unique(f)) == {0.0, 5.0}
    j, i = np.nonzero(f)
    assert np.all(np.abs(i / 23 - 0.3) <= 0.1) and np.all(np.abs(j / 23 - 0.6) <= 0.1)
    assert not forcing_plane(3).any()
