"""The ensemble batch (BASELINE config 5) undamped and globalised, measured.
    python tools/ens_globalized_bench.py [--K 8192] [--reps 3]

bench.py's ensemble inputs (`bench.ensemble_params`, K = 8192 trajectories of the 2D Brusselator at N = 32, GMRES with
modified Gram-Schmidt, abstol 1e-8), four algorithms: NewtonRaphson; TrustRegion with the Simple and with the NLsolve radius
scheme; NewtonRaphson with BackTracking.  Each runs from the reference u0 and from 10 u0 + 0.1.  Per arm: problems/s from
CUDA events over `reps` timed solves after one warm-up solve, successes and the retcode histogram, the worst residual, Newton
steps and Arnoldi iterations per Newton step, and the solve kernel's resident CTAs per SM from the occupancy query.  The
ensemble API reports no per-step trace, so rejected and backtracked steps are not counted.

From 10 u0 + 0.1 GMRES can outgrow the default 512-column basis slab, and such trajectories are redone one by one by the
general driver.  Those arms therefore run with B200_ENS_BASIS_COLUMNS = n (2048 columns: 8.6 GB of slabs at two CTAs per SM)
on the first --K-far trajectories (default 1024; the Arnoldi work per trajectory is several times that of a solve from u0).  Progress goes to stderr; one JSON line, with the card, its power
limit and its maximum SM clock, goes to stdout."""
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
ALGS = (
    ("newton_raphson", lambda: nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(orth="mgs"))),
    ("trust_region_simple", lambda: nls.TrustRegion(linsolve=nls.KrylovJL_GMRES(orth="mgs"), radius_update_scheme=nls.RadiusUpdateSchemes.Simple)),
    ("trust_region_nlsolve", lambda: nls.TrustRegion(linsolve=nls.KrylovJL_GMRES(orth="mgs"), radius_update_scheme=nls.RadiusUpdateSchemes.NLsolve)),
    ("backtracking", lambda: nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(orth="mgs"), linesearch=nls.BackTracking())),
)


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def run_arm(ctx, stream, K, reps, alg, d_u0, d_A, d_B):
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
    rc, counts = np.unique(cache.rc.to_host(), return_counts=True)
    return {"problems_per_s": K / (ms * 1e-3), "ms_median": ms, "ms_all": [round(t, 2) for t in times], "n_success": int(res.nsuccess),
            "retcodes": {nls.ReturnCode.name(int(r)): int(c) for r, c in zip(rc, counts)}, "worst_resid_inf": res.worst_resid_inf,
            "newton_steps": int(res.total_nsteps), "max_newton_steps": int(res.max_nsteps), "arnoldi_iters": int(res.total_njvp),
            "arnoldi_iters_per_newton_step": res.total_njvp / max(1, res.total_nsteps), "ctas_per_sm": cache.ctas_per_sm()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--K", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--K-far", dest="K_far", type=int, default=1024)
    args = ap.parse_args()
    assert args.reps >= 3
    torch.cuda.init()
    ctx = nls.Context(0)
    stream = torch.cuda.current_stream()
    K = args.K
    A, B = bench.ensemble_params(K)
    dp = nls._DeviceProblem(ctx, nls.NonlinearProblem(nls.Brusselator2D(N), None, (3.4, 1.0, ALPHA), ctx=ctx))
    u = dp.u0().to_host()
    arms = {}
    for start, u0, k in (("u0", u, K), ("10u0+0.1", 10.0 * u + 0.1, min(K, args.K_far))):
        if start != "u0":
            os.environ["B200_ENS_BASIS_COLUMNS"] = str(2 * N * N)
        d_u0, d_A, d_B = ctx.to_device(np.tile(u0, k)), ctx.to_device(A[:k]), ctx.to_device(B[:k])
        for name, make in ALGS:
            key = "%s@%s" % (name, start)
            arms[key] = run_arm(ctx, stream, k, args.reps, make(), d_u0, d_A, d_B)
            arms[key]["K"] = k
            print(key, json.dumps(arms[key]), file=sys.stderr, flush=True)
        base = arms["newton_raphson@%s" % start]["problems_per_s"]
        for name, _ in ALGS:
            arms["%s@%s" % (name, start)]["rate_vs_newton_raphson"] = arms["%s@%s" % (name, start)]["problems_per_s"] / base
    os.environ.pop("B200_ENS_BASIS_COLUMNS", None)
    print(json.dumps({"tool": "ens_globalized_bench", "workload": "ensemble_bruss2d_N%d_gmres_mgs_abstol1e-8" % N, "K": K, "K_far": min(K, args.K_far),
                      "card": card(), "arms": arms}))


if __name__ == "__main__":
    main()
