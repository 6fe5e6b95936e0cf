"""The resident Arnoldi kernel's global tail at the benchmarked size (3D Brusselator N = 100): bit for bit the same results
whichever way the tail pairs travel.

At N = 100 on an H100 the shared-memory stages hold qs = 21 of each thread's 30 row pairs; the other 9 are copied by cp.async
into stage slots the thread has released (csrc/gmres.cu, R3_SLOTGET; tests/test_resident_tail_slots.py restates the slot map).
B200_RESIDENT_STAGE_PAIRS caps qs, which moves the kernel between its paths with the same arithmetic in the same order:
  21  the stock split: every tail pair from a slot;
  12  slots for pairs 12 .. 20 (update sweeps) and 12 .. 23 (dot sweeps), the rest straight from global memory;
   9  the smallest split whose update sweeps still copy their tail (R3_TAIL_AT); the copy is waited for at once;
   5  update sweeps read their tail from global memory, dot sweeps use 5 slots;
   1  one slot per dot sweep, every other tail pair from global memory.
Each configuration runs once, matrix-free and on the assembled sparse Jacobian, with MGS and with the reorthogonalised
variant (which wraps around into a second Gram-Schmidt pass every step)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ENV = "B200_RESIDENT_STAGE_PAIRS"
N = 100
ITMAX = 40
CAPS = (21, 12, 9, 5, 1)


@pytest.fixture(scope="module")
def problem(nls, ctx, po):
    f, P = nls.Brusselator3D(N), po.OracleProblem.bruss3d(N)
    dp = nls._DeviceProblem(ctx, nls.NonlinearProblem(f, None, (3.4, 1.0, 10.0), ctx=ctx))
    u = P.u0(1)
    return P, dp, ctx.to_device(u), ctx.to_device(P.residual(u))


def _solve(nls, ctx, n, A, b, orth):
    cnt = ITMAX * (ITMAX + 3) // 2
    gm = nls.GmresSolver(ctx, n, nls.KrylovJL_GMRES(orth=orth, engine="resident", itmax=ITMAX), atol=1e-8, rtol=3e-13, keep_hessenberg=cnt)
    x, st = gm.solve(A, b)
    return st.iters, st.rnorm, gm.hessenberg(st.iters), x.to_host()


@pytest.mark.parametrize("orth", ["mgs", "cgs2"])
@pytest.mark.parametrize("opkind", ["matrix-free", "assembled"])
def test_tail_paths_are_bit_identical_at_n100(nls, ctx, problem, monkeypatch, orth, opkind):
    P, dp, u, b = problem
    assert ctx.sm_count() * 7680 >= N ** 3 > ctx.sm_count() * 21 * 256    # a global tail exists at the stock split
    if opkind == "assembled":
        sj = nls.SparseJacobian(dp)
        A = ("sparse_jac", sj, sj.fill(u))
    else:
        A = nls.JacobianOperator(dp, u)
    monkeypatch.delenv(ENV, raising=False)
    ref = _solve(nls, ctx, P.n, A, b, orth)
    assert ref[0] == ITMAX
    for cap in CAPS:
        monkeypatch.setenv(ENV, str(cap))
        got = _solve(nls, ctx, P.n, A, b, orth)
        what = "cap %d, %s, %s" % (cap, orth, opkind)
        assert got[0] == ref[0] and got[1] == ref[1], (what, got[:2], ref[:2])
        assert np.array_equal(got[2], ref[2]), (what, "Hessenberg", np.flatnonzero(got[2] != ref[2])[:5])
        assert np.array_equal(got[3], ref[3]), (what, "x", np.abs(got[3] - ref[3]).max())
