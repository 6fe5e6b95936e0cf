"""The ensemble batch (BASELINE config 5) with and without the multigrid preconditioner, measured.
    python tools/ens_precond_bench.py [--K 8192] [--reps 3]

bench.py's ensemble inputs (`bench.ensemble_params`, K = 8192 trajectories of the 2D Brusselator at N = 32 from the reference
u0, GMRES with modified Gram-Schmidt, abstol 1e-8), four ways: no preconditioner; Multigrid("right") with the inherited GMRES
tolerances; Multigrid("left") with atol 1e-13, rtol 1e-9 (left preconditioning tests the preconditioned residual, so it sets
the Krylov tolerances itself); Multigrid("right") with EisenstatWalkerForcing2.  Per arm: problems/s from CUDA events over
`reps` timed solves after one warm-up solve, successes, the worst residual, mean Arnoldi iterations per Newton step, and the
solve kernel's resident CTAs per SM from the occupancy query.  Prints one JSON line, with the card, its power limit and its
maximum SM clock."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import nonlinearsolve_jl_b200 as nls  # noqa: E402

N, ALPHA = 32, 10.0
ARMS = (
    ("none", dict(), None),
    ("multigrid_right", dict(precs=nls.Multigrid("right")), None),
    ("multigrid_left", dict(precs=nls.Multigrid("left"), atol=1e-13, rtol=1e-9), None),
    ("multigrid_right_ew", dict(precs=nls.Multigrid("right")), nls.EisenstatWalkerForcing2()),
)


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def run_arm(ctx, stream, K, reps, gm, forcing, d_u0, d_A, d_B):
    alg = nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(orth="mgs", **gm), forcing=forcing)
    cache = nls.EnsembleCache(ctx, N, K, ALPHA, alg, abstol=1e-8)
    res = cache.solve(d_u0, d_A, d_B)  # warm-up: workspace allocation, module load
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        res = cache.solve(d_u0, d_A, d_B)
        e1.record(stream)
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    ms = float(np.median(times))
    return {"problems_per_s": K / (ms * 1e-3), "ms_median": ms, "ms_all": [round(t, 2) for t in times], "n_success": int(res.nsuccess),
            "worst_resid_inf": res.worst_resid_inf, "newton_steps": int(res.total_nsteps), "arnoldi_iters": int(res.total_njvp),
            "arnoldi_iters_per_newton_step": res.total_njvp / max(1, res.total_nsteps), "ctas_per_sm": cache.ctas_per_sm()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--K", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    assert args.reps >= 3
    torch.cuda.init()
    ctx = nls.Context(0)
    stream = torch.cuda.current_stream()
    K = args.K
    A, B = bench.ensemble_params(K)
    dp = nls._DeviceProblem(ctx, nls.NonlinearProblem(nls.Brusselator2D(N), None, (3.4, 1.0, ALPHA), ctx=ctx))
    d_u0, d_A, d_B = ctx.to_device(np.tile(dp.u0().to_host(), K)), ctx.to_device(A), ctx.to_device(B)
    arms = {name: run_arm(ctx, stream, K, args.reps, gm, forcing, d_u0, d_A, d_B) for name, gm, forcing in ARMS}
    base = arms["none"]["problems_per_s"]
    for a in arms.values():
        a["speedup_vs_none"] = a["problems_per_s"] / base
    print(json.dumps({"tool": "ens_precond_bench", "workload": "ensemble_%d_x_bruss2d_N%d_newtonraphson_gmres_mgs" % (K, N), "card": card(),
                      "arms": arms}))


if __name__ == "__main__":
    main()
