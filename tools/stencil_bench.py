"""Stand-alone K1 / K2 timing (residual f(u), JVP J(u)v, VJP) at N = 100 / 80 on operands that do NOT sit in L2: the kernels cycle
over SETS buffer triples (SETS * 3 * Bv > 400 MB, far above the 50 MB L2).  Two clocks: the library's per-launch CUDA events (ctx.profile) and the wall
clock around a back-to-back batch (launch overhead included).   python tools/stencil_bench.py [N ...]
Algorithmic bytes: residual 2 Bv (+ the N^2 forcing plane), JVP / VJP 3 Bv."""
import json
import sys
import time
sys.path.insert(0, ".")
import numpy as np  # noqa: E402
import nonlinearsolve_jl_b200 as nls  # noqa: E402

PEAK = json.load(open("MEASURED_PEAKS.json")).get("hbm_gbs", 3350.0) if __import__("os").path.exists("MEASURED_PEAKS.json") else 3350.0
ctx = nls.Context(0)
out = {}
for N in [int(a) for a in sys.argv[1:]] or [100, 80]:
    f = nls.Brusselator3D(N)
    dp = nls._DeviceProblem(ctx, nls.NonlinearProblem(f, None, (3.4, 1.0, 10.0), ctx=ctx))
    n = dp.n
    Bv = 8.0 * n
    SETS = max(4, int(400e6 / (3 * Bv)) + 1)
    rng = np.random.default_rng(N)
    us = [ctx.to_device(dp.u0(1).to_host() + 0.01 * rng.standard_normal(n)) for _ in range(SETS)]
    vs = [ctx.to_device(rng.standard_normal(n)) for _ in range(SETS)]
    os_ = [ctx.empty(n) for _ in range(SETS)]
    res = {}
    for name, call, nb in (("residual", lambda s: dp.residual(us[s], os_[s]), 2.0), ("jvp", lambda s: dp.jvp(us[s], vs[s], os_[s]), 3.0),
                           ("vjp", lambda s: dp.vjp(us[s], vs[s], os_[s]), 3.0)):
        for s in range(SETS):
            call(s)
        ctx.sync()
        ctx.profile(True)
        reps = 5 * SETS
        for r in range(reps):
            call(r % SETS)
        ctx.sync()
        rep = ctx.profile_report()
        ctx.profile(False)
        fam = rep["residual" if name == "residual" else "jvp"]
        ev_us = fam["ms"] * 1e3 / fam["launches"]
        t0 = time.perf_counter()
        for r in range(reps):
            call(r % SETS)
        ctx.sync()
        wall_us = (time.perf_counter() - t0) * 1e6 / reps
        res[name] = {"bytes": nb * Bv, "event_us": round(ev_us, 2), "event_gbs": round(nb * Bv / ev_us / 1e3, 1), "event_frac": round(nb * Bv / ev_us / 1e3 / PEAK, 3),
                     "batch_wall_us": round(wall_us, 2), "batch_gbs": round(nb * Bv / wall_us / 1e3, 1)}
    # the ceiling for kernels this short: the library's plain copy kernel (2 Bv of traffic) through the same harness
    import ctypes as C
    cp = lambda s: nls.abi.check(ctx.handle, nls.abi.lib().b200_copy(ctx.handle, C.c_int64(n), us[s].ptr, os_[s].ptr))  # noqa: E731
    for s in range(SETS):
        cp(s)
    ctx.sync()
    t0 = time.perf_counter()
    for r in range(5 * SETS):
        cp(r % SETS)
    ctx.sync()
    wall_us = (time.perf_counter() - t0) * 1e6 / (5 * SETS)
    res["copy_2Bv"] = {"bytes": 2 * Bv, "batch_wall_us": round(wall_us, 2), "batch_gbs": round(2 * Bv / wall_us / 1e3, 1)}
    out["N%d" % N] = res
print(json.dumps(out, indent=1))
