"""GPU: cost of the resident Arnoldi kernel's global-memory tail, one row pair per thread at a time.

    python tools/resident_tail_sweep.py [itmax] [mgs|cgs2]

At N = 100 a CTA owns 15 152 rows (30 row pairs per thread) and the shared-memory stages hold the first `qs` of them; the
other 30 - qs pairs of the two shared-memory-role vectors are read from global memory.  The tools/resident_phases.py workload
(one GMRES solve of `itmax` iterations, resident engine) is timed at the stock split and with B200_RESIDENT_STAGE_PAIRS
capping the stages at 18, 15, 12 and 9 pairs, three repetitions each, then at N = 80 (every row on chip) once.  The slope of
us per basis vector against tail pairs per thread is the cost of one tail pair per vector."""
import json
import os
import subprocess
import sys
import time
sys.path.insert(0, ".")
import nonlinearsolve_jl_b200 as nls  # noqa: E402

ITMAX = int(sys.argv[1]) if len(sys.argv) > 1 else 300
ORTH = sys.argv[2] if len(sys.argv) > 2 else "mgs"
PASSES = 1 if ORTH == "mgs" else 2
CAPS = (None, 18, 15, 12, 9)  # None: the stock split
STOCK_QS = (232448 - 14 * 256 * 16 - 2048) // 8192  # gm_resident_plan's rule on the H100's 227 KB of opt-in shared memory: 21
ctx = nls.Context(0)


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], stdout=subprocess.PIPE, text=True)
    return r.stdout.strip()


def us_per_vector(N, reps):
    f = nls.Brusselator3D(N)
    dp = nls._DeviceProblem(ctx, nls.NonlinearProblem(f, None, (3.4, 1.0, 10.0), ctx=ctx))
    u = dp.u0(1); b = dp.residual(u)
    gm = nls.GmresSolver(ctx, dp.n, nls.KrylovJL_GMRES(orth=ORTH, engine="resident", itmax=ITMAX), atol=0.0, rtol=1e-14)
    gm.solve(nls.JacobianOperator(dp, u), b)  # warm-up
    out = []
    for _ in range(reps):
        ctx.sync(); t = time.time()
        gm.solve(nls.JacobianOperator(dp, u), b)
        ctx.sync(); dt = time.time() - t
        out.append(dt * 1e6 / (PASSES * ITMAX * (ITMAX + 1) / 2))
    del gm
    return out


def tail_pairs(N, qs):
    """largest number of global-memory row pairs of a thread: rows per CTA over 512, rounded up, minus the stage's pairs"""
    G = ctx.sm_count()
    nc = N ** 3
    cpc = (nc + G - 1) // G
    cpc += cpc & 1
    pairs = min(30, -(-2 * cpc // 512))
    return max(0, pairs - qs)


rows = []
print(json.dumps({"card": card(), "orth": ORTH, "itmax": ITMAX}))
for cap in CAPS:
    if cap is None:
        os.environ.pop("B200_RESIDENT_STAGE_PAIRS", None)
    else:
        os.environ["B200_RESIDENT_STAGE_PAIRS"] = str(cap)
    us = us_per_vector(100, 3)
    rows.append({"N": 100, "cap": cap, "tail_pairs": tail_pairs(100, STOCK_QS if cap is None else cap), "us_per_vector": [round(x, 3) for x in us]})
    print(json.dumps(rows[-1]), flush=True)
os.environ.pop("B200_RESIDENT_STAGE_PAIRS", None)
rows.append({"N": 80, "cap": None, "tail_pairs": 0, "us_per_vector": [round(x, 3) for x in us_per_vector(80, 1)]})
print(json.dumps(rows[-1]), flush=True)
# least-squares slope of the median us per vector against tail pairs (N = 100 rows)
pts = [(r["tail_pairs"], sorted(r["us_per_vector"])[1]) for r in rows if r["N"] == 100]
mx = sum(x for x, _ in pts) / len(pts); my = sum(y for _, y in pts) / len(pts)
slope = sum((x - mx) * (y - my) for x, y in pts) / sum((x - mx) ** 2 for x, _ in pts)
print(json.dumps({"slope_us_per_tail_pair": round(slope, 4), "stock_us_per_vector": pts[0][1], "stock_tail_pairs": pts[0][0],
                  "tail_share_at_stock": round(slope * pts[0][0] / pts[0][1], 3)}))
