"""Ruge-Stueben and smoothed-aggregation AMG as the `precs` of GMRES on the sparse route, measured.
    python tools/amg_bench.py [--skip-config4]

Config 4 exactly as bench.py's sparse_tr leg sets it up (3D Brusselator N = 100, coloured sparse Jacobian, TrustRegion, GMRES
with modified Gram-Schmidt on the assembled matrix), six ways: no preconditioner, ILU0("left"), RugeStubenAMG("left" / "right")
and SmoothedAggregationAMG("left" / "right").  Then each AMG alone on config 4's Jacobian at u0: the hierarchy (unknowns and
nonzeros per level, operator complexity, device bytes it holds), the rebuild, the refresh, and one V-cycle with its bytes/s
against the algorithmic bytes defined in `cycle_bytes`.  Last, a user residual with a jac_prototype (2D N = 128 periodic
diffusion with a cubic reaction, evaluated by torch) with and without AMG, where the same per-hierarchy numbers are taken on
the Jacobian at u0.  Prints one JSON line, with the card and its power limit."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import nonlinearsolve_jl_b200 as nls  # noqa: E402

# Left preconditioning makes GMRES test the preconditioned residual, so the left variants set the Krylov tolerances themselves
# (as the project's tests do); the right variant keeps the unpreconditioned run's inherited tolerances.
LEFT = dict(atol=1e-13, rtol=1e-9)
VARIANTS = (("none", dict()), ("ilu0_left", dict(precs=nls.ILU0("left"), **LEFT)), ("amg_left", dict(precs=nls.RugeStubenAMG("left"), **LEFT)),
            ("amg_right", dict(precs=nls.RugeStubenAMG("right"))), ("sa_left", dict(precs=nls.SmoothedAggregationAMG("left"), **LEFT)),
            ("sa_right", dict(precs=nls.SmoothedAggregationAMG("right"))))
METHODS = (("amg", nls.SparseAMG), ("sa", nls.SparseAMG.smoothed_aggregation))


def timed(stream, fn, reps=1, warm=1):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    out = None
    for _ in range(reps):
        out = fn()
    e1.record(stream)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, out


def summary(ms, sol):
    steps = max(1, sol.stats.nsteps)
    return {"s_per_solve": ms * 1e-3, "newton_steps": sol.stats.nsteps, "njacs": sol.stats.njacs,
            "arnoldi_iters_per_step": sum(t.lin_iters for t in sol.trace) / steps, "resid_inf": sol.resid_inf,
            "retcode": nls.ReturnCode.name(sol.retcode)}


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def cycle_bytes(amg, ns, nzs):
    """Algorithmic bytes of one V(nu1, nu2) cycle: on every level but the coarsest, each pass over A (the residual and the
    nu1 - 1 + nu2 Jacobi sweeps) moves nnz * 12 (value + int32 column) plus four vectors (x, b, 1/diag, result); R r and
    P x_c each move P's nnz * 12 plus a fine and a coarse vector (the prolongation also reads and writes x); the first
    pre-sweep moves three vectors; the coarsest level moves its dense inverse and two vectors."""
    o = amg.opts
    total = 0.0
    for l in range(len(ns) - 1):
        pnnz = int(amg._export(l, nls.abi.AMG_EXPORT_P, ns[l])[2][-1])
        sweeps = max(o.presweeps - 1, 0) + 1 + o.postsweeps
        total += sweeps * (12.0 * nzs[l] + 4 * 8.0 * ns[l])
        total += (24.0 * ns[l] if o.presweeps > 0 else 8.0 * ns[l])
        total += 12.0 * pnnz + 8.0 * (ns[l] + ns[l + 1])            # restriction
        total += 12.0 * pnnz + 8.0 * (2 * ns[l] + ns[l + 1])        # prolongation-add
    total += 8.0 * ns[-1] * ns[-1] + 16.0 * ns[-1]
    return total


def hierarchy(ctx, stream, make, n, sj, nz):
    """One AMG alone on the Jacobian values nz: levels, device bytes, rebuild, refresh and one V-cycle."""
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    amg = make(ctx, n, sj.colptr, sj.rowval, 1)
    t0 = time.perf_counter()
    rebuild_ms, info = timed(stream, lambda: amg.setup(nz, rebuild=True), warm=0)
    rebuild_wall_s = time.perf_counter() - t0
    free1 = torch.cuda.mem_get_info()[0]
    rebuild2_ms, _ = timed(stream, lambda: amg.setup(nz, rebuild=True), warm=0)
    refresh_ms, info2 = timed(stream, lambda: amg.setup(nz, rebuild=False), reps=3)
    b = ctx.to_device(np.random.default_rng(0).standard_normal(n))
    x = ctx.zeros(n)
    apply_ms, _ = timed(stream, lambda: amg.solve(b, x), reps=20, warm=2)
    ns, nzs = amg.levels()
    nbytes = cycle_bytes(amg, ns, nzs)
    out = {"nnz": sj.nnz, "levels_n": ns, "levels_nnz": nzs, "operator_complexity": sum(nzs) / nzs[0], "setup_info": [info, info2],
           "device_bytes_held": free0 - free1, "rebuild_ms": [rebuild_ms, rebuild2_ms], "rebuild_wall_s": rebuild_wall_s, "refresh_ms": refresh_ms,
           "apply_ms": apply_ms, "apply_bytes": nbytes, "apply_GBps": nbytes / (apply_ms * 1e-3) / 1e9}
    del amg
    torch.cuda.empty_cache()
    return out


def config4(ctx, stream):
    N = 100
    f = nls.Brusselator3D(N)
    dp = nls._DeviceProblem(ctx, nls.NonlinearProblem(f, None, (3.4, 1.0, 10.0), ctx=ctx))
    u0 = dp.u0(nls.abi.U0_PERTURBED_Z)
    out = {"workload": "bruss3d_N100_trustregion_sparse_jacobian_gmres", "unknowns": dp.n}
    sj = nls.SparseJacobian(dp)
    nz = sj.fill(u0)
    for key, make in METHODS:
        out[key] = hierarchy(ctx, stream, make, dp.n, sj, nz)
    del sj, nz
    torch.cuda.empty_cache()
    fs = nls.NonlinearFunction(f, sparsity=nls.TracerSparsityDetector())
    for name, kw in VARIANTS:
        cache = nls.init(nls.NonlinearProblem(fs, u0, (3.4, 1.0, 10.0), ctx=ctx), nls.TrustRegion(linsolve=nls.KrylovJL_GMRES(orth="mgs", **kw)), abstol=1e-8)

        def step():
            cache.reinit(u0)
            return cache.solve(to_host=False)
        ms, sol = timed(stream, step)
        out[name] = summary(ms, sol)
        del cache
        torch.cuda.empty_cache()
    return out


def user_problem(ctx, stream, N=128):
    n = N * N
    a = 0.25 * N * N

    def lap(x):
        g = x.view(N, N)
        return (4.0 * g - g.roll(1, 0) - g.roll(-1, 0) - g.roll(1, 1) - g.roll(-1, 1)).reshape(-1)

    def F(du, u, _p):
        du_t, u_t = torch.as_tensor(du, device="cuda"), torch.as_tensor(u, device="cuda")
        du_t.copy_(a * lap(u_t) + u_t ** 3 - 1.0)
        torch.cuda.synchronize()

    def JVP(Jv, v, u, _p):
        Jv_t, v_t, u_t = (torch.as_tensor(y, device="cuda") for y in (Jv, v, u))
        Jv_t.copy_(a * lap(v_t) + 3.0 * u_t * u_t * v_t)
        torch.cuda.synchronize()

    colptr, rowval = [1], []
    for c in range(n):
        i, j = c % N, c // N
        rowval.extend(r + 1 for r in sorted({c, (i + 1) % N + N * j, (i - 1) % N + N * j, i + N * ((j + 1) % N), i + N * ((j - 1) % N)}))
        colptr.append(len(rowval) + 1)
    fn = nls.NonlinearFunction(F, jvp=JVP, n=n, jac_prototype=(np.array(colptr, dtype=np.int64), np.array(rowval, dtype=np.int64), 1))
    u0 = 0.5 + 0.1 * np.sin(np.arange(n))
    out = {"workload": "user_callback_2d_N%d_jac_prototype_newtonraphson_sparse_gmres" % N, "unknowns": n}
    dp = nls._DeviceProblem(ctx, nls.NonlinearProblem(fn, u0, None, ctx=ctx))
    sj = nls.SparseJacobian(dp)
    nz = sj.fill(ctx.to_device(u0))
    for key, make in METHODS:
        out[key] = hierarchy(ctx, stream, make, n, sj, nz)
    del dp, sj, nz
    for name, kw in (VARIANTS[0],) + VARIANTS[2:]:
        prob = nls.NonlinearProblem(fn, u0, None, ctx=ctx)
        alg = nls.NewtonRaphson(linsolve=nls.KrylovJL_GMRES(**kw))
        ms, sol = timed(stream, lambda: nls.solve(prob, alg, abstol=1e-9), reps=3)
        out[name] = summary(ms, sol)
    return out


def main():
    # a stream of its own (the legacy default stream would make the context create another one): the library's work and the
    # timing events share it
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    ctx = nls.Context(0, stream=stream.cuda_stream)
    line = {"card": card()}
    if "--skip-config4" not in sys.argv:
        line["config4"] = config4(ctx, stream)
    line["user_2d"] = user_problem(ctx, stream)
    line["card_after"] = card()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
