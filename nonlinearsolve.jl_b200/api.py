"""Host-side mirror of the reference's interface for the first-order Newton path, over the C ABI.

Names, argument meaning and error behaviour follow NonlinearSolve.jl so that the parity tests read like the
reference's own tests:

    prob = NonlinearProblem(Brusselator3D(100), u0, (3.4, 1.0, 10.0))
    sol  = solve(prob, NewtonRaphson(linsolve=KrylovJL_GMRES()), abstol=1e-8)
    sol.u, sol.resid, sol.retcode, sol.stats.nsteps

Reference: NewtonRaphson lib/NonlinearSolveFirstOrder/src/raphson.jl:30-43, TrustRegion trust_region.jl:25-43,
solve/init/step!/solve!/reinit! lib/NonlinearSolveBase/src/solve.jl:76-442, 835-858, NLStats usage solve.jl:142,
JacobianOperator lib/SciMLJacobianOperators/src/SciMLJacobianOperators.jl:86-243, EnsembleProblem usage
test/PolyAlgorithms/core_tests__item6.jl:3-20.  In the real drop-in these classes are Julia structs in
julia/B200Newton issuing the same C calls (INTEGRATION.md); Python is the executable harness in this environment.

Everything here runs on the GPU through libb200newton.so.  There is no CPU path.
"""
import ctypes as C
import weakref

import numpy as np

from . import _abi as abi
from ._abi import check, lib


# ----------------------------------------------------------------------------- context / device memory
def _destroy_context(handle, children):
    for fin in reversed(children):
        fin()  # idempotent: a finalizer that already ran is a no-op
    children.clear()
    lib().b200_ctx_destroy(handle)


class Context:
    """One CUDA device + stream + library workspaces (b200_ctx).  Not thread-safe (one per host thread)."""

    def __init__(self, device=0, stream=None):
        self._h = C.c_void_p()
        st = lib().b200_ctx_create(int(device), C.c_void_p(stream) if stream else None, C.byref(self._h))
        if st == abi.ERR_NO_DEVICE:
            raise abi.B200Error(st, "no CUDA device available: the B200 backend has no CPU fallback")
        if st != abi.OK:
            raise abi.B200Error(st, "b200_ctx_create failed")
        self.device = device
        self._children = []  # finalizers of every library object created on this context
        self._fin = weakref.finalize(self, _destroy_context, self._h, self._children)

    @property
    def handle(self):
        return self._h

    def _adopt(self, fin):
        """Register a child object's finalizer: whatever the garbage collector's order, the context destroys every
        object created on it (newest first) before it destroys itself, so no child ever runs against a dead context."""
        ch = self._children
        ch.append(fin)
        if len(ch) > 4096:
            ch[:] = [f for f in ch if f.alive]
        return fin

    def sync(self):
        check(self._h, lib().b200_ctx_sync(self._h))

    @property
    def stream(self):
        return lib().b200_ctx_stream(self._h)

    def kernel_launches(self):
        n = C.c_int64(0)
        check(self._h, lib().b200_ctx_kernel_launches(self._h, C.byref(n)))
        return n.value

    def sm_count(self):
        n = C.c_int32(0)
        check(self._h, lib().b200_ctx_sm_count(self._h, C.byref(n)))
        return n.value

    def flush_l2(self):
        check(self._h, lib().b200_flush_l2(self._h))

    def profile(self, on=True, reset=True):
        """Enable/disable per-kernel-family CUDA-event timing on the context stream."""
        if reset:
            check(self._h, lib().b200_ctx_profile_reset(self._h))
        check(self._h, lib().b200_ctx_profile_enable(self._h, 1 if on else 0))

    def profile_report(self):
        """{family: {"ms", "bytes", "launches", "gbs"}} accumulated since the last reset."""
        out = {}
        for kid, name in enumerate(abi.KID_NAMES):
            ms, by, ln = C.c_double(), C.c_double(), C.c_int64()
            check(self._h, lib().b200_ctx_profile_get(self._h, kid, C.byref(ms), C.byref(by), C.byref(ln)))
            if ln.value:
                out[name] = {"ms": ms.value, "bytes": by.value, "launches": ln.value,
                             "gbs": (by.value / (ms.value * 1e-3) / 1e9) if ms.value > 0 else 0.0}
        return out

    def pinned_empty(self, n, dtype=np.float64):
        """A NumPy view of pinned host memory (b200_host_alloc) for the end-to-end host-buffer path."""
        dt = np.dtype(dtype)
        p = C.c_void_p()
        check(self._h, lib().b200_host_alloc(self._h, int(n) * dt.itemsize, C.byref(p)))
        buf = (C.c_char * (int(n) * dt.itemsize)).from_address(p.value)
        arr = np.frombuffer(buf, dtype=dt)
        self._pinned = getattr(self, "_pinned", [])
        self._pinned.append((p, buf))
        return arr

    # memory
    def empty(self, n, dtype=np.float64):
        return DeviceVector(self, int(n), dtype)

    def zeros(self, n, dtype=np.float64):
        v = DeviceVector(self, int(n), dtype)
        check(self._h, lib().b200_memset(self._h, v.ptr, 0, v.nbytes))
        return v

    def to_device(self, arr, dtype=None):
        arr = np.ascontiguousarray(arr, dtype=dtype or np.asarray(arr).dtype)
        v = DeviceVector(self, arr.size, arr.dtype)
        v.copy_from_host(arr)
        return v


def device_count():
    """Number of CUDA devices the library sees (0 without a GPU; the library never falls back to the CPU)."""
    n = C.c_int32(0)
    lib().b200_device_count(C.byref(n))
    return n.value


_default_ctx = {}


def default_context(device=0):
    """Lazily created per-device context (the Julia glue keeps one per task)."""
    if device not in _default_ctx:
        _default_ctx[device] = Context(device)
    return _default_ctx[device]


class DeviceVector:
    """A device buffer owned by the library allocator (b5: the array type handed to the solver instead of CuArray)."""

    def __init__(self, ctx, n, dtype=np.float64, ptr=None, owner=None):
        self.ctx, self.n, self.dtype = ctx, int(n), np.dtype(dtype)
        self.nbytes = self.n * self.dtype.itemsize
        self._owner = owner
        if ptr is None:
            p = C.c_void_p()
            check(ctx.handle, lib().b200_malloc(ctx.handle, max(self.nbytes, 16), C.byref(p)))
            self.ptr = p
            self._fin = ctx._adopt(weakref.finalize(self, lib().b200_free, ctx.handle, p))
        else:
            self.ptr = C.c_void_p(ptr if isinstance(ptr, int) else ptr.value)

    def __len__(self):
        return self.n

    def view(self, offset, n):
        return DeviceVector(self.ctx, n, self.dtype, ptr=self.ptr.value + offset * self.dtype.itemsize, owner=self)

    def copy_from_host(self, arr):
        arr = np.ascontiguousarray(arr, dtype=self.dtype)
        assert arr.size == self.n
        check(self.ctx.handle, lib().b200_memcpy_h2d(self.ctx.handle, self.ptr, arr.ctypes.data_as(C.c_void_p), self.nbytes))
        return self

    def to_host(self):
        out = np.empty(self.n, dtype=self.dtype)
        check(self.ctx.handle, lib().b200_memcpy_d2h(self.ctx.handle, out.ctypes.data_as(C.c_void_p), self.ptr, self.nbytes))
        return out

    def copy(self):
        v = DeviceVector(self.ctx, self.n, self.dtype)
        check(self.ctx.handle, lib().b200_memcpy_d2d(self.ctx.handle, v.ptr, self.ptr, self.nbytes))
        return v

    @property
    def __cuda_array_interface__(self):
        return {"shape": (self.n,), "typestr": self.dtype.str, "data": (self.ptr.value, False), "version": 3}

    # the BLAS-1 surface L2-L4 of the reference touch on a device array (SURVEY.md §8b, b5)
    def norm(self, p=2):
        out = C.c_double()
        fn = lib().b200_nrm2 if p == 2 else lib().b200_norminf
        check(self.ctx.handle, fn(self.ctx.handle, self.n, self.ptr, C.byref(out)))
        return out.value

    def dot(self, other):
        out = C.c_double()
        check(self.ctx.handle, lib().b200_dot(self.ctx.handle, self.n, self.ptr, other.ptr, C.byref(out)))
        return out.value

    def axpy(self, a, x):  # self += a x
        check(self.ctx.handle, lib().b200_axpy(self.ctx.handle, self.n, float(a), x.ptr, self.ptr))
        return self

    def scal(self, a):
        check(self.ctx.handle, lib().b200_scal(self.ctx.handle, self.n, float(a), self.ptr))
        return self

    def fill(self, a):
        check(self.ctx.handle, lib().b200_fill(self.ctx.handle, self.n, float(a), self.ptr))
        return self


def _as_device(ctx, x):
    if isinstance(x, DeviceVector):
        return x
    return ctx.to_device(np.asarray(x, dtype=np.float64).ravel(order="F"))


# ----------------------------------------------------------------------------- return codes / stats / solution
class ReturnCode:
    Default, Success, MaxIters, MaxTime, Stalled, StalledSuccess, Unstable = 0, 1, 2, 3, 4, 5, 6
    InternalLinearSolveFailed, InternalLineSearchFailed, ShrinkThresholdExceeded, InitialFailure, Failure = 7, 8, 9, 10, 11
    ConvergenceFailure = 12

    @staticmethod
    def name(code):
        return abi.RETCODE_NAMES.get(int(code), "Unknown")


def successful_retcode(code):
    """SciMLBase.successful_retcode."""
    return int(code) in (ReturnCode.Success, ReturnCode.StalledSuccess)


class NLStats:
    """SciMLBase.NLStats(nf, njacs, nfactors, nsolve, nsteps) (+ njvp, an extension)."""

    def __init__(self, nf=0, njacs=0, nfactors=0, nsolve=0, nsteps=0, njvp=0):
        self.nf, self.njacs, self.nfactors, self.nsolve, self.nsteps, self.njvp = nf, njacs, nfactors, nsolve, nsteps, njvp

    def __repr__(self):
        return "NLStats(nf=%d, njacs=%d, nfactors=%d, nsolve=%d, nsteps=%d, njvp=%d)" % (
            self.nf, self.njacs, self.nfactors, self.nsolve, self.nsteps, self.njvp)


class NonlinearSolution:
    def __init__(self, prob, alg, u, resid, retcode, stats, trace=None, bytes_moved=0.0, resid_inf=None):
        self.prob, self.alg, self.u, self.resid, self.retcode, self.stats, self.trace = prob, alg, u, resid, retcode, stats, trace
        self.bytes_moved = bytes_moved
        self.resid_inf = resid_inf

    def __repr__(self):
        return "NonlinearSolution(retcode=%s, %r)" % (ReturnCode.name(self.retcode), self.stats)


# ----------------------------------------------------------------------------- user functions / problems
class _BuiltinFunction:
    """A residual whose f!/jvp!/vjp!/jac! are the library's fused kernels (what a Julia user would get by passing
    `NonlinearFunction(B200Newton.brusselator!(...); jvp = ..., jac_prototype = ...)`)."""
    kind = None
    has_pattern = True

    def n(self):
        raise NotImplementedError


class Brusselator2D(_BuiltinFunction):
    """brusselator_2d_loop of sparsity_tests__item1.jl:13-36; p = (A, B, alpha) with dx = 1/(N-1) implied."""
    kind = abi.PROB_BRUSS2D

    def __init__(self, N):
        self.N = int(N)

    def n(self):
        return 2 * self.N * self.N

    def default_p(self):
        return (3.4, 1.0, 10.0)


class Brusselator3D(Brusselator2D):
    """3D extension (SURVEY.md §A.2)."""
    kind = abi.PROB_BRUSS3D

    def n(self):
        return 2 * self.N ** 3


class QuadraticFunction(_BuiltinFunction):
    """quadratic_f(u, p) = u .* u .- p  (common/common_rootfind_testing.jl:15)."""
    kind = abi.PROB_QUADRATIC

    def __init__(self, n):
        self._n = int(n)

    def n(self):
        return self._n

    def default_p(self):
        return 2.0


class TridiagQuadFunction(_BuiltinFunction):
    """F(u, p) = u + 0.1 u .* (T u) - p with T = Tridiagonal(-1, 2, -1)  (rootfind_tests__item20.jl:6-29)."""
    kind = abi.PROB_TRIDIAG_QUAD

    def __init__(self, n):
        self._n = int(n)

    def n(self):
        return self._n


class NonlinearFunction:
    """NonlinearFunction{true}(f!; jvp = jvp!, vjp = vjp!, sparsity = ..., jac_prototype = ..., colorvec = ...).

    `f` is either one of the built-in device functions above or a Python callable `f(du, u, p)` whose arguments arrive as
    objects exposing `__cuda_array_interface__` (wrap with torch.as_tensor(x, device="cuda")); the callable must enqueue
    its work on the context's stream or finish before returning.  `jvp(Jv, v, u, p)`, `vjp(Jtw, w, u, p)` likewise.
    """

    def __init__(self, f, jvp=None, vjp=None, sparsity=None, jac_prototype=None, colorvec=None, n=None, jac=None):
        self.f, self.jvp, self.vjp = f, jvp, vjp
        # jac(J, u, p): fills the concrete Jacobian in place (b3; jacobian.jl:241-243).  J arrives as a DeviceVector over the
        # dense column-major n*n matrix, or over `nzval` when jac_prototype = (colptr, rowval) describes a CSC pattern.
        self.jac = jac
        self.sparsity, self.jac_prototype, self.colorvec = sparsity, jac_prototype, colorvec
        self._n = n

    @property
    def builtin(self):
        return isinstance(self.f, _BuiltinFunction)


class TracerSparsityDetector:
    """Marker: use the structural pattern (ADTypes sparsity detector role, jacobian.jl:286-353)."""


class NonlinearProblem:
    def __init__(self, f, u0, p=None, ctx=None):
        self.f = f if isinstance(f, NonlinearFunction) else NonlinearFunction(f)
        self.u0 = u0
        self.p = p
        self.ctx = ctx


def remake(prob, u0=None, p=None):
    return NonlinearProblem(prob.f, prob.u0 if u0 is None else u0, prob.p if p is None else p, prob.ctx)


# ----------------------------------------------------------------------------- algorithms
class KrylovJL_GMRES:
    """LinearSolve.KrylovJL_GMRES(; gmres_restart = 0, ...) -> Krylov.gmres!  (restart off, memory 20, MGS).

    `orth` selects the Gram-Schmidt variant of the device engine: "mgs" (Krylov.jl default), "cgs", "cgs2"
    (Krylov's `reorthogonalization = true` analogue; the default here because it is the robust one at 1e-8)."""

    needs_concrete_A = False

    def __init__(self, gmres_restart=0, memory=20, itmax=0, orth="cgs2", warm_start=False, atol=None, rtol=None, check_every=None,
                 engine="auto", block=0, precs=None):
        # precs: LinearSolve's `precs = (A, p) -> (Pl, Pr)`; here a BlockJacobi(side) descriptor of the built-in preconditioner
        self.precs = precs
        self.block = 0      # reserved (the L2-blocked Gram-Schmidt of round 1 was slower than the streaming kernels and is gone)
        self.gmres_restart, self.memory, self.itmax, self.orth = gmres_restart, memory, itmax, orth
        self.warm_start, self.atol, self.rtol, self.check_every, self.engine = warm_start, atol, rtol, check_every, engine

    def fill(self, g):
        g.memory, g.restart, g.itmax = int(self.memory), int(self.gmres_restart), int(self.itmax)
        g.orth = {"mgs": abi.ORTH_MGS, "cgs": abi.ORTH_CGS, "cgs2": abi.ORTH_CGS2}[self.orth]
        g.warm_start = 1 if self.warm_start else 0
        g.engine = {"auto": abi.ENGINE_AUTO, "multikernel": abi.ENGINE_MULTIKERNEL, "resident": abi.ENGINE_RESIDENT}[self.engine]
        g.check_every = int(self.check_every) if self.check_every is not None else 0  # 0: the library's default (8; 2 with a preconditioner)
        g.block = int(self.block)
        g.atol = float(self.atol) if self.atol is not None else 0.0
        g.rtol = float(self.rtol) if self.rtol is not None else 0.0


class BlockJacobi:
    """Built-in preconditioner for `KrylovJL_GMRES(precs = ...)`: the inverse of the 2x2 species blocks on the diagonal of
    the Brusselator Jacobian, rebuilt from the current iterate at every Newton step (what `precs(A, p)` returning
    `(Pl, I)` or `(I, Pr)` does in the reference, test/Core/core_tests__item21.jl)."""

    def __init__(self, side="left"):
        assert side in ("left", "right")
        self.side = side

    @property
    def code(self):
        return abi.PRECOND_BLOCK_JACOBI_LEFT if self.side == "left" else abi.PRECOND_BLOCK_JACOBI_RIGHT

    def linop(self, dprob, u):
        """A borrowed-by-GMRES operator handle applying the inverse at iterate u (DeviceVector)."""
        op = C.c_void_p()
        check(dprob.ctx.handle, lib().b200_linop_block_jacobi(dprob.handle, u.ptr, C.byref(op)))
        return op


class Multigrid:
    """Built-in preconditioner for `KrylovJL_GMRES(precs = ...)`: one geometric-multigrid V-cycle of the Brusselator Jacobian
    (coarsening by the prime factors of N down to one cell, damped block-Jacobi smoothing), rebuilt from the current iterate
    at every Newton step — the role `AlgebraicMultigrid.aspreconditioner(ruge_stuben(W))` plays in
    docs/src/tutorials/large_systems.md:290-316."""

    def __init__(self, side="right"):
        assert side in ("left", "right")
        self.side = side

    @property
    def code(self):
        return abi.PRECOND_MULTIGRID_LEFT if self.side == "left" else abi.PRECOND_MULTIGRID_RIGHT

    def linop(self, dprob, u):
        op = C.c_void_p()
        check(dprob.ctx.handle, lib().b200_linop_precond(dprob.handle, u.ptr, self.code, C.byref(op)))
        return op


class ILU0:
    """Preconditioner for `KrylovJL_GMRES(precs = ...)` on the concrete sparse Jacobian: the incomplete LU with zero fill of
    the assembled J, refactorised with every fresh Jacobian — the first `precs` of docs/src/tutorials/large_systems.md:244-316
    (`IncompleteLU.ilu(W, τ = 50.0)` there; here no threshold, the pattern of J).  Needs `concrete_jac = True` or a sparse
    prototype, and serves any problem with a pattern, including a user residual with `jac_prototype`."""

    def __init__(self, side="left"):
        assert side in ("left", "right")
        self.side = side

    @property
    def code(self):
        return abi.PRECOND_ILU0_LEFT if self.side == "left" else abi.PRECOND_ILU0_RIGHT


class RugeStubenAMG:
    """Preconditioner for `KrylovJL_GMRES(precs = ...)` on the concrete sparse Jacobian: one classical Ruge-Stueben algebraic
    multigrid V-cycle with damped Jacobi smoothing — the tutorial's `AlgebraicMultigrid.aspreconditioner(ruge_stuben(W))` with
    Jacobi smoothers (docs/src/tutorials/large_systems.md:244-316), default options (theta 0.25, omega 2/3, V(1,1)).  The
    splitting is chosen at the first fresh Jacobian of a solve; later Jacobians refresh every value on the device.  Needs
    `concrete_jac = True` or a sparse prototype, and serves any problem with a pattern, including `jac_prototype`."""

    def __init__(self, side="left"):
        assert side in ("left", "right")
        self.side = side

    @property
    def code(self):
        return abi.PRECOND_AMG_LEFT if self.side == "left" else abi.PRECOND_AMG_RIGHT


class SmoothedAggregationAMG:
    """Preconditioner for `KrylovJL_GMRES(precs = ...)` on the concrete sparse Jacobian: one smoothed-aggregation algebraic
    multigrid V-cycle with damped Jacobi smoothing — the tutorial's `AlgebraicMultigrid.aspreconditioner(smoothed_aggregation(W))`
    with Jacobi smoothers (docs/src/tutorials/large_systems.md:244-316), default options (theta 0.08, omega 2/3, V(1,1),
    smooth_omega 4/3).  The aggregates are chosen on the device at the first fresh Jacobian of a solve; later Jacobians refresh
    every value.  Needs `concrete_jac = True` or a sparse prototype, and serves any problem with a pattern."""

    def __init__(self, side="left"):
        assert side in ("left", "right")
        self.side = side

    @property
    def code(self):
        return abi.PRECOND_SA_AMG_LEFT if self.side == "left" else abi.PRECOND_SA_AMG_RIGHT


class LUFactorization:
    needs_concrete_A = True


class KLUFactorization:
    """LinearSolve.KLUFactorization(): sparse direct factorisation of the concrete sparse Jacobian (operator_jacobian.jl:22).
    Device route: reverse Cuthill-McKee + banded LU with partial pivoting (b200_sparse_lu_*)."""
    needs_concrete_A = True


UMFPACKFactorization = KLUFactorization


class SparseBandLU:
    """Direct handle on the device sparse direct solver for a CSC pattern (colptr, rowval host arrays, 1-based by default)."""

    def __init__(self, ctx, n, colptr, rowval, index_base=1):
        self.ctx, self.n = ctx, n
        colptr = np.ascontiguousarray(colptr, dtype=np.int64)
        rowval = np.ascontiguousarray(rowval, dtype=np.int64)
        self._h = C.c_void_p()
        check(ctx.handle, lib().b200_sparse_lu_create(ctx.handle, n, colptr.ctypes.data_as(C.c_void_p), rowval.ctypes.data_as(C.c_void_p), index_base, C.byref(self._h)))
        self._fin = ctx._adopt(weakref.finalize(self, lib().b200_sparse_lu_destroy, self._h))

    def bandwidth(self):
        kl, ku = C.c_int64(0), C.c_int64(0)
        check(self.ctx.handle, lib().b200_sparse_lu_bandwidth(self._h, C.byref(kl), C.byref(ku)))
        return kl.value, ku.value

    def factor(self, nzval):
        info = C.c_int32(0)
        check(self.ctx.handle, lib().b200_sparse_lu_factor(self._h, nzval.ptr, C.byref(info)))
        return info.value

    def solve(self, b, x=None):
        x = x or self.ctx.zeros(self.n)
        check(self.ctx.handle, lib().b200_sparse_lu_solve(self._h, b.ptr, x.ptr))
        return x


class SparseILU0:
    """Direct handle on the device ILU(0) of a CSC pattern (colptr, rowval host arrays, 1-based by default): `factor(nzval)`
    returns 0 or the 1-based row of a zero / non-finite pivot, `solve(b)` applies U^-1 L^-1, `factors()` returns the packed
    factors in the pattern's CSC order (L strictly below the diagonal, unit diagonal implied; U on and above it)."""

    def __init__(self, ctx, n, colptr, rowval, index_base=1):
        self.ctx, self.n = ctx, n
        colptr = np.ascontiguousarray(colptr, dtype=np.int64)
        rowval = np.ascontiguousarray(rowval, dtype=np.int64)
        self.nnz = int(colptr[n] - colptr[0])
        self._h = C.c_void_p()
        check(ctx.handle, lib().b200_ilu0_create(ctx.handle, n, colptr.ctypes.data_as(C.c_void_p), rowval.ctypes.data_as(C.c_void_p), index_base, C.byref(self._h)))
        self._fin = ctx._adopt(weakref.finalize(self, lib().b200_ilu0_destroy, self._h))

    def levels(self):
        lo, up = C.c_int32(0), C.c_int32(0)
        check(self.ctx.handle, lib().b200_ilu0_levels(self._h, C.byref(lo), C.byref(up)))
        return lo.value, up.value

    def factor(self, nzval):
        info = C.c_int32(0)
        check(self.ctx.handle, lib().b200_ilu0_factor(self._h, nzval.ptr, C.byref(info)))
        return info.value

    def solve(self, b, x=None):
        x = x or self.ctx.zeros(self.n)
        check(self.ctx.handle, lib().b200_ilu0_solve(self._h, b.ptr, x.ptr))
        return x

    def factors(self, out=None):
        out = out or self.ctx.zeros(self.nnz)
        check(self.ctx.handle, lib().b200_ilu0_export(self._h, out.ptr))
        return out

    def linop(self):
        """A borrowed-by-GMRES operator handle applying U^-1 L^-1 (destroy it with b200_linop_destroy before this handle)."""
        op = C.c_void_p()
        check(self.ctx.handle, lib().b200_ilu0_linop(self._h, C.byref(op)))
        return op


class SparseAMG:
    """Direct handle on the device Ruge-Stueben hierarchy of a CSC pattern (colptr, rowval host arrays, 1-based by default), or
    with `SparseAMG.smoothed_aggregation(...)` the smoothed-aggregation one.
    Options: theta, omega, presweeps, postsweeps, max_levels, max_coarse (b200_amg_opts; b200_sa_opts adds smooth_omega).
    `setup(nzval, rebuild=True)` returns 0 or the 1-based level of a zero diagonal / pivot (rebuild=False keeps the splitting or
    the aggregates and recomputes the values), `solve(b)` applies one V-cycle, `levels()` returns the unknowns and nonzeros per
    level, `level(l)` the CSR arrays of A_l and P_l (and of the tentative prolongator T_l on smoothed-aggregation handles)."""

    def __init__(self, ctx, n, colptr, rowval, index_base=1, _method="ruge_stuben", **opts):
        self.ctx, self.n = ctx, n
        self.method = _method
        colptr = np.ascontiguousarray(colptr, dtype=np.int64)
        rowval = np.ascontiguousarray(rowval, dtype=np.int64)
        sa = _method == "smoothed_aggregation"
        o = abi.SaOpts() if sa else abi.AmgOpts()
        (lib().b200_sa_opts_default if sa else lib().b200_amg_opts_default)(C.byref(o))
        for k, v in opts.items():
            assert k in dict(o._fields_), k
            setattr(o, k, v)
        self.opts = o
        self._h = C.c_void_p()
        create = lib().b200_amg_create_sa if sa else lib().b200_amg_create
        check(ctx.handle, create(ctx.handle, n, colptr.ctypes.data_as(C.c_void_p), rowval.ctypes.data_as(C.c_void_p), index_base, C.byref(o),
                                 C.byref(self._h)))
        self._fin = ctx._adopt(weakref.finalize(self, lib().b200_amg_destroy, self._h))

    @classmethod
    def smoothed_aggregation(cls, ctx, n, colptr, rowval, index_base=1, **opts):
        """The smoothed-aggregation hierarchy (b200_amg_create_sa): options theta, omega, presweeps, postsweeps, max_levels,
        max_coarse, smooth_omega."""
        return cls(ctx, n, colptr, rowval, index_base, _method="smoothed_aggregation", **opts)

    def setup(self, nzval, rebuild=True):
        info = C.c_int32(0)
        check(self.ctx.handle, lib().b200_amg_setup(self._h, nzval.ptr, int(bool(rebuild)), C.byref(info)))
        return info.value

    def solve(self, b, x=None):
        x = x or self.ctx.zeros(self.n)
        check(self.ctx.handle, lib().b200_amg_solve(self._h, b.ptr, x.ptr))
        return x

    def levels(self):
        cap = 64
        nl = C.c_int32(0)
        ns, nz = np.zeros(cap, dtype=np.int64), np.zeros(cap, dtype=np.int64)
        check(self.ctx.handle, lib().b200_amg_levels(self._h, C.byref(nl), ns.ctypes.data_as(C.c_void_p), nz.ctypes.data_as(C.c_void_p), cap))
        return ns[:nl.value].tolist(), nz[:nl.value].tolist()

    def _export(self, level, what, nrows):
        rowptr = np.zeros(nrows + 1, dtype=np.int32)
        check(self.ctx.handle, lib().b200_amg_export(self._h, level, what, rowptr.ctypes.data_as(C.c_void_p), None, None))
        col = np.zeros(int(rowptr[-1]), dtype=np.int32)
        val = np.zeros(int(rowptr[-1]), dtype=np.float64)
        check(self.ctx.handle, lib().b200_amg_export(self._h, level, what, rowptr.ctypes.data_as(C.c_void_p), col.ctypes.data_as(C.c_void_p),
                                                     val.ctypes.data_as(C.c_void_p)))
        return val, col, rowptr

    def level(self, l):
        """{"A": (data, indices, indptr), "P": ... or None on the coarsest level}: `scipy.sparse.csr_matrix(level["A"])` builds A_l.
        Smoothed-aggregation handles add "T", the tentative prolongator (None on the coarsest level)."""
        ns, _ = self.levels()
        out = {"A": self._export(l, abi.AMG_EXPORT_A, ns[l]), "P": None}
        if l + 1 < len(ns):
            out["P"] = self._export(l, abi.AMG_EXPORT_P, ns[l])
        if self.method == "smoothed_aggregation":
            out["T"] = self._export(l, abi.AMG_EXPORT_T, ns[l]) if l + 1 < len(ns) else None
        return out

    def linop(self):
        """A borrowed-by-GMRES operator handle applying one V-cycle (destroy it with b200_linop_destroy before this handle)."""
        op = C.c_void_p()
        check(self.ctx.handle, lib().b200_amg_linop(self._h, C.byref(op)))
        return op


def amg_split(n, colptr, rowval, nzval, index_base=1, theta=0.25):
    """The level-0 Ruge-Stueben C/F splitting on the host (no device): (boolean array, True at C points; number of C points)."""
    colptr = np.ascontiguousarray(colptr, dtype=np.int64)
    rowval = np.ascontiguousarray(rowval, dtype=np.int64)
    nzval = np.ascontiguousarray(nzval, dtype=np.float64)
    cf = np.zeros(n, dtype=np.int32)
    nc = C.c_int64()
    st = lib().b200_amg_split(n, colptr.ctypes.data_as(C.c_void_p), rowval.ctypes.data_as(C.c_void_p), nzval.ctypes.data_as(C.c_void_p), index_base,
                              theta, cf.ctypes.data_as(C.c_void_p), C.byref(nc))
    if st != abi.OK:
        raise abi.B200Error(st, "b200_amg_split failed")
    return cf.astype(bool), nc.value


class AutoForwardDiff:
    jvp_mode = abi.JVP_EXACT


class AutoFiniteDiff:
    jvp_mode = abi.JVP_FINITE_DIFF


class EisenstatWalkerForcing2:
    """eisenstat_walker.jl:18-30."""

    def __init__(self, eta0=0.5, eta_max=0.9, gamma=0.9, alpha=2.0, safeguard=True, safeguard_threshold=0.1):
        self.eta0, self.eta_max, self.gamma, self.alpha = eta0, eta_max, gamma, alpha
        self.safeguard, self.safeguard_threshold = safeguard, safeguard_threshold


class _TerminationMode:
    """Termination modes of NonlinearSolveBase (public.jl:300-407).  `norm`: the mode's internalnorm — "inf" (maximum(abs, .),
    the NonlinearProblem default) or "l2" (norm(., 2)); Safe modes take `max_stalled_steps` (None: no step-norm stall test,
    as when the reference's constructor is called without it; the solver's own default mode uses 32)."""
    code = abi.TERM_ABS_NORM_SAFE_BEST
    safe = False

    def __init__(self, norm="inf", max_stalled_steps=32):
        assert norm in ("inf", "l2")
        self.norm = abi.NORM_INF if norm == "inf" else abi.NORM_L2
        self.max_stalled_steps = -1 if (max_stalled_steps is None or not self.safe) else int(max_stalled_steps)


class AbsNormSafeBestTerminationMode(_TerminationMode):
    code, safe = abi.TERM_ABS_NORM_SAFE_BEST, True


class AbsNormSafeTerminationMode(_TerminationMode):
    code, safe = abi.TERM_ABS_NORM_SAFE, True


class AbsNormTerminationMode(_TerminationMode):
    code = abi.TERM_ABS_NORM


class NormTerminationMode(_TerminationMode):
    code = abi.TERM_NORM


class RelTerminationMode(_TerminationMode):
    code = abi.TERM_REL


class RelNormTerminationMode(_TerminationMode):
    code = abi.TERM_REL_NORM


class AbsTerminationMode(_TerminationMode):
    code = abi.TERM_ABS


class RelNormSafeTerminationMode(_TerminationMode):
    code, safe = abi.TERM_REL_NORM_SAFE, True


class RelNormSafeBestTerminationMode(_TerminationMode):
    code, safe = abi.TERM_REL_NORM_SAFE_BEST, True


class BackTracking:
    """LineSearch.BackTracking(; c_1 = 1e-4, rho_hi = 0.5, rho_lo = 0.1, maxiters = 1000), cubic interpolation."""

    def __init__(self, c_1=1e-4, rho_hi=0.5, rho_lo=0.1, maxiters=1000):
        self.c_1, self.rho_hi, self.rho_lo, self.maxiters = c_1, rho_hi, rho_lo, maxiters


class _FirstOrder:
    name = "GeneralizedFirstOrderAlgorithm"
    globalization = abi.GLOB_NONE

    def __init__(self, concrete_jac=None, linsolve=None, autodiff=None, jvp_autodiff=None, vjp_autodiff=None, forcing=None, linesearch=None):
        self.concrete_jac, self.linsolve, self.autodiff = concrete_jac, linsolve, autodiff
        self.jvp_autodiff, self.vjp_autodiff, self.forcing = jvp_autodiff, vjp_autodiff, forcing
        self.linesearch = linesearch


class NewtonRaphson(_FirstOrder):
    """NewtonRaphson(; concrete_jac, linsolve, autodiff, jvp_autodiff, vjp_autodiff, forcing)  raphson.jl:30-43."""
    name = "NewtonRaphson"


class PseudoTransient(_FirstOrder):
    """PseudoTransient(; alpha_initial = 1e-3, linsolve, linesearch, ...): DampedNewtonDescent with switched evolution
    relaxation, (J + I/alpha) du = -f, alpha_{n+1} = alpha_n ||f_{n-1}|| / ||f_n||  (pseudo_transient.jl:37-56, 157-170)."""
    name = "PseudoTransient"
    descent = abi.DESCENT_PSEUDO_TRANSIENT

    def __init__(self, concrete_jac=None, linsolve=None, autodiff=None, jvp_autodiff=None, vjp_autodiff=None, linesearch=None, alpha_initial=1.0e-3):
        super().__init__(concrete_jac, linsolve, autodiff, jvp_autodiff, vjp_autodiff, None, linesearch)
        self.alpha_initial = float(alpha_initial)


class LevenbergMarquardt(_FirstOrder):
    """LevenbergMarquardt(; damping_initial = 1.0, α_geodesic = 0.75, disable_geodesic = Val(false), damping_increase_factor = 2.0,
    damping_decrease_factor = 3.0, finite_diff_step_geodesic = 0.1, b_uphill = 1.0, min_damping_D = 1e-8)
    (levenberg_marquardt.jl:36-61): damped normal equations with the running-maximum diagonal, geodesic acceleration, and the
    uphill-accepting trust region; concrete dense Jacobian.  The trace's `trust_radius` slot carries the damping λ used by the
    step, `lin_status` the geodesic-acceleration verdict."""
    name = "LevenbergMarquardt"
    descent = abi.DESCENT_LEVENBERG_MARQUARDT

    def __init__(self, damping_initial=1.0, alpha_geodesic=0.75, disable_geodesic=False, damping_increase_factor=2.0, damping_decrease_factor=3.0,
                 finite_diff_step_geodesic=0.1, b_uphill=1.0, min_damping_D=1e-8, autodiff=None):
        super().__init__(True, None, autodiff, None, None, None, None)
        self.lm = dict(lm_damping_initial=damping_initial, lm_alpha_geodesic=alpha_geodesic, lm_damping_increase=damping_increase_factor,
                       lm_damping_decrease=damping_decrease_factor, lm_finite_diff_step=finite_diff_step_geodesic,
                       lm_b_uphill=(b_uphill if b_uphill > 0 else -1.0), lm_min_damping_D=min_damping_D)
        self.disable_geodesic = bool(disable_geodesic)


class Broyden(_FirstOrder):
    """Broyden(; max_resets = 100, reset_tolerance = nothing, init_jacobian = Val(:identity), alpha = nothing, update_rule =
    Val(:good_broyden))  NonlinearSolveQuasiNewton/src/broyden.jl:34-51 — the quasi-Newton family's dense Broyden (SURVEY §8f-4):
    NewtonDescent on a stored inverse that stays in HBM, rank-one update per step, NoChangeInStateReset, ConvergenceFailure after
    `max_resets`.  `init_jacobian`: "identity" | "true_jacobian"; `update_rule`: "good_broyden" | "bad_broyden".  The trace's
    `lin_status` slot flags the steps before which J^-1 was re-initialised."""
    name = "Broyden"
    descent = abi.DESCENT_BROYDEN

    def __init__(self, max_resets=100, reset_tolerance=None, init_jacobian="identity", alpha=None, update_rule="good_broyden", autodiff=None):
        init_jacobian, update_rule = str(init_jacobian).strip(":"), str(update_rule).strip(":")
        if init_jacobian not in ("identity", "true_jacobian"):
            raise ValueError("Unknown `init_jacobian = %r`: identity or true_jacobian" % init_jacobian)
        if update_rule not in ("good_broyden", "bad_broyden"):
            raise ValueError("Unknown update rule %r: good_broyden or bad_broyden (the diagonal structure is not offered)" % update_rule)
        super().__init__(init_jacobian == "true_jacobian", None, autodiff, None, None, None, None)
        self.qn = dict(qn_init_jacobian=abi.QN_INIT_TRUE_JACOBIAN if init_jacobian == "true_jacobian" else abi.QN_INIT_IDENTITY,
                       qn_update_rule=abi.QN_UPDATE_BAD_BROYDEN if update_rule == "bad_broyden" else abi.QN_UPDATE_GOOD_BROYDEN,
                       qn_max_resets=int(max_resets))
        self.reset_tolerance, self.alpha = reset_tolerance, alpha


class LimitedMemoryBroyden(Broyden):
    """LimitedMemoryBroyden(; max_resets = 3, threshold = Val(10), reset_tolerance = nothing, alpha = nothing)
    NonlinearSolveQuasiNewton/src/lbroyden.jl:20-35 — good Broyden on J^-1 = alpha I + U V' with the last `threshold` updates kept
    (two n x threshold arrays): the member of the family that scales to the 2*10^6-unknown systems."""
    name = "LimitedMemoryBroyden"

    def __init__(self, max_resets=3, threshold=10, reset_tolerance=None, alpha=None):
        super().__init__(max_resets=max_resets, reset_tolerance=reset_tolerance, init_jacobian="identity", alpha=alpha)
        self.qn["qn_init_jacobian"] = abi.QN_INIT_LOW_RANK
        self.qn["qn_threshold"] = int(threshold)


class Klement(Broyden):
    """Klement(; max_resets = 100, alpha = nothing, init_jacobian = Val(:identity))  NonlinearSolveQuasiNewton/src/klement.jl:30-49 — with
    the default initialisation the approximate Jacobian has the DIAGONAL structure: an n-vector, elementwise descent and update, any n.
    (`init_jacobian = true_jacobian / true_jacobian_diagonal` are not offered.)"""
    name = "Klement"

    def __init__(self, max_resets=100, alpha=None):
        super().__init__(max_resets=max_resets, init_jacobian="identity", alpha=alpha)
        self.qn["qn_update_rule"] = abi.QN_UPDATE_KLEMENT


class RadiusUpdateSchemes:
    """RadiusUpdateSchemes.{Simple, NLsolve, NocedalWright, Hei, Yuan, Fan, Bastin}  (trust_region.jl:431-520)."""
    Simple, NLsolve, NocedalWright, Hei, Yuan, Fan, Bastin = (abi.TR_SIMPLE, abi.TR_NLSOLVE, abi.TR_NOCEDAL_WRIGHT, abi.TR_HEI, abi.TR_YUAN, abi.TR_FAN, abi.TR_BASTIN)


class TrustRegion(_FirstOrder):
    """TrustRegion(; radius_update_scheme = RadiusUpdateSchemes.Simple, ...) with Dogleg descent  trust_region.jl:25-43.
    Thresholds / factors left at `None` (or 0) take the scheme's defaults (trust_region.jl:330-384)."""
    name = "TrustRegion"
    globalization = abi.GLOB_TRUST_REGION

    def __init__(self, concrete_jac=None, linsolve=None, autodiff=None, jvp_autodiff=None, vjp_autodiff=None, max_trust_radius=0.0,
                 initial_trust_radius=0.0, step_threshold=None, shrink_threshold=None, expand_threshold=None, shrink_factor=None,
                 expand_factor=None, max_shrink_times=32, radius_update_scheme=abi.TR_SIMPLE):
        super().__init__(concrete_jac, linsolve, autodiff, jvp_autodiff, vjp_autodiff, None)
        self.radius_update_scheme = int(radius_update_scheme)
        step_threshold, shrink_threshold, expand_threshold, shrink_factor, expand_factor = (
            0.0 if v is None else v for v in (step_threshold, shrink_threshold, expand_threshold, shrink_factor, expand_factor))
        self.tr = dict(tr_max_trust_radius=max_trust_radius, tr_initial_trust_radius=initial_trust_radius,
                       tr_step_threshold=step_threshold, tr_shrink_threshold=shrink_threshold, tr_expand_threshold=expand_threshold,
                       tr_shrink_factor=shrink_factor, tr_expand_factor=expand_factor)
        self.max_shrink_times = max_shrink_times


def _build_opts(prob, alg, abstol, reltol, maxiters, termination_condition, store_trace, maxtime=None):
    o = abi.NewtonOpts()
    lib().b200_newton_opts_default(C.byref(o))
    o.abstol = float(abstol) if abstol is not None else 0.0
    o.reltol = float(reltol) if reltol is not None else 0.0
    o.maxiters = int(maxiters)
    o.store_trace = 1 if store_trace else 0
    o.globalization = alg.globalization
    o.descent = getattr(alg, "descent", abi.DESCENT_NEWTON)
    o.pt_alpha_initial = getattr(alg, "alpha_initial", 0.0)
    o.maxtime = float(maxtime) if maxtime is not None else 0.0
    if termination_condition is not None:
        if isinstance(termination_condition, type):
            termination_condition = termination_condition()
        o.termination = termination_condition.code
        o.term_norm = termination_condition.norm
        o.term_max_stalled_steps = termination_condition.max_stalled_steps
    ls = alg.linsolve
    sparse = prob.f.sparsity is not None or prob.f.jac_prototype is not None
    if ls is None or isinstance(ls, (LUFactorization, KLUFactorization)):
        # linsolve === nothing -> LinearSolve default: dense LU for a dense J, a sparse direct factorisation (KLU / UMFPACK)
        # for a sparse J (sparsity_tests__item1.jl:54-93).  Device route for the latter: RCM + banded LU (b200_sparse_lu_*);
        # at sizes whose band does not fit (3D N = 100) newton_create fails with B200_ERR_NOMEM and the message says to use
        # `linsolve = KrylovJL_GMRES()` on the assembled matrix, which is what the reference's own GPU test does
        # (test/gpu/cuda_tests__item1.jl:32).
        if isinstance(ls, KLUFactorization) and not sparse:
            raise TypeError("KLUFactorization needs a sparse Jacobian (sparsity / jac_prototype)")
        o.linsolve = abi.LINSOLVE_SPARSE_LU if sparse else abi.LINSOLVE_DENSE_LU
    elif isinstance(ls, KrylovJL_GMRES):
        ls.fill(o.gmres)
        if getattr(ls, "precs", None) is not None:
            o.precond = ls.precs.code
        if alg.concrete_jac or sparse:  # needs_concrete_A false but concrete_jac = Val(true)  (jacobian.jl:43-47)
            o.linsolve = abi.LINSOLVE_SPARSE_GMRES
        else:
            o.linsolve = abi.LINSOLVE_GMRES
    else:
        raise TypeError("unsupported linsolve %r" % (ls,))
    ad = alg.jvp_autodiff or alg.autodiff
    if ad is not None:
        o.jvp_mode = ad.jvp_mode
    if alg.forcing is not None:
        f = alg.forcing
        o.forcing = abi.FORCING_EW2
        o.ew_eta0, o.ew_eta_max, o.ew_gamma, o.ew_alpha = f.eta0, f.eta_max, f.gamma, f.alpha
        o.ew_safeguard, o.ew_safeguard_threshold = (1 if f.safeguard else 0), f.safeguard_threshold
    ls_ = getattr(alg, "linesearch", None)
    if ls_ is not None:  # has_linesearch (solve.jl:249-273): globalization = Val(:LineSearch)
        o.globalization = abi.GLOB_LINESEARCH
        o.ls_c1, o.ls_rho_hi, o.ls_rho_lo, o.ls_maxiters = float(ls_.c_1), float(ls_.rho_hi), float(ls_.rho_lo), int(ls_.maxiters)
    if isinstance(alg, LevenbergMarquardt):
        if sparse:
            raise TypeError("LevenbergMarquardt is offered on the dense concrete Jacobian")
        o.linsolve = abi.LINSOLVE_DENSE_LU
        for k, v in alg.lm.items():
            setattr(o, k, float(v))
        o.lm_disable_geodesic = 1 if alg.disable_geodesic else 0
    if isinstance(alg, Broyden):
        if sparse:
            raise TypeError("Broyden keeps a dense inverse: no sparse prototype")
        # the stored inverse needs no linear solver; the dense LU is there only to invert the true Jacobian at (re)initialisation
        o.linsolve = abi.LINSOLVE_DENSE_LU if alg.qn["qn_init_jacobian"] == abi.QN_INIT_TRUE_JACOBIAN else abi.LINSOLVE_GMRES
        for k, v in alg.qn.items():
            setattr(o, k, int(v))
        o.qn_reset_tolerance = float(alg.reset_tolerance) if alg.reset_tolerance is not None else 0.0
        o.qn_alpha = float(alg.alpha) if alg.alpha is not None else 0.0
    if isinstance(alg, TrustRegion):
        for k, v in alg.tr.items():
            setattr(o, k, float(v))
        o.max_shrink_times = int(alg.max_shrink_times)
        o.tr_scheme = int(alg.radius_update_scheme)
    return o


class _DeviceProblem:
    """Owns the b200_problem handle for a NonlinearProblem (built-in kernels or host callbacks)."""

    def __init__(self, ctx, prob):
        self.ctx = ctx
        self._h = C.c_void_p()
        self._keep = []
        f = prob.f
        L = lib()
        if f.builtin:
            fn = f.f
            p = prob.p if prob.p is not None else getattr(fn, "default_p", lambda: None)()
            if fn.kind in (abi.PROB_BRUSS2D, abi.PROB_BRUSS3D):
                A, B, alpha = (float(x) for x in p[:3])
                if len(p) > 3:  # the reference passes dx = step(range(0, 1, length = N)) as p[4]
                    assert abs(p[3] - 1.0 / (fn.N - 1)) < 1e-15, "dx must be 1/(N-1) as in the reference problem"
                create = L.b200_problem_create_bruss2d if fn.kind == abi.PROB_BRUSS2D else L.b200_problem_create_bruss3d
                check(ctx.handle, create(ctx.handle, fn.N, A, B, alpha, C.byref(self._h)))
            elif fn.kind == abi.PROB_QUADRATIC:
                check(ctx.handle, L.b200_problem_create_quadratic(ctx.handle, fn.n(), float(p), C.byref(self._h)))
            elif fn.kind == abi.PROB_TRIDIAG_QUAD:
                pv = _as_device(ctx, p)
                self._keep.append(pv)
                check(ctx.handle, L.b200_problem_create_tridiag_quad(ctx.handle, fn.n(), pv.ptr, C.byref(self._h)))
                ctx.sync()
            self.n = fn.n()
        else:
            n = f._n if f._n is not None else int(np.asarray(prob.u0).size if not isinstance(prob.u0, DeviceVector) else prob.u0.n)
            self.n = n
            pp = prob.p

            def wrap(ptr):
                return DeviceVector(ctx, n, np.float64, ptr=ptr)

            def f_cb(user, u, du):
                try:
                    f.f(wrap(du), wrap(u), pp)
                    return 0
                except Exception:  # noqa: BLE001 - no exception may cross the ABI
                    import traceback
                    traceback.print_exc()
                    return 1

            def jvp_cb(user, u, v, Jv):
                try:
                    f.jvp(wrap(Jv), wrap(v), wrap(u), pp)
                    return 0
                except Exception:  # noqa: BLE001
                    import traceback
                    traceback.print_exc()
                    return 1

            def vjp_cb(user, u, w, Jtw):
                try:
                    f.vjp(wrap(Jtw), wrap(w), wrap(u), pp)
                    return 0
                except Exception:  # noqa: BLE001
                    import traceback
                    traceback.print_exc()
                    return 1

            self._f_cb = abi.RESIDUAL_CB(f_cb)
            self._jvp_cb = abi.JVP_CB(jvp_cb) if f.jvp is not None else C.cast(None, abi.JVP_CB)
            self._vjp_cb = abi.JVP_CB(vjp_cb) if f.vjp is not None else C.cast(None, abi.JVP_CB)
            check(ctx.handle, L.b200_problem_create_callback(ctx.handle, n, self._f_cb, self._jvp_cb, self._vjp_cb, None, C.byref(self._h)))
        self._jac_cb = None
        if isinstance(f.jac_prototype, tuple):  # jac_prototype = (colptr, rowval[, index_base]) : CSC structure of J0
            cp = np.ascontiguousarray(f.jac_prototype[0], dtype=np.int64)
            rv = np.ascontiguousarray(f.jac_prototype[1], dtype=np.int64)
            base = int(f.jac_prototype[2]) if len(f.jac_prototype) > 2 else 1
            check(ctx.handle, L.b200_problem_set_jac_prototype(self._h, cp.ctypes.data_as(C.c_void_p), rv.ctypes.data_as(C.c_void_p), base))
        if f.jac is not None:
            sparse_proto = f.jac_prototype is not None or f.sparsity is not None
            pp_, n_ = prob.p, self.n

            def jac_cb(user, u, J):
                try:
                    cnt = self._jac_len if sparse_proto else n_ * n_
                    f.jac(DeviceVector(ctx, cnt, np.float64, ptr=J), DeviceVector(ctx, n_, np.float64, ptr=u), pp_)
                    return 0
                except Exception:  # noqa: BLE001 - no exception may cross the ABI
                    import traceback
                    traceback.print_exc()
                    return 1
            self._jac_len = len(f.jac_prototype[1]) if isinstance(f.jac_prototype, tuple) else 0
            self._jac_cb = abi.JAC_CB(jac_cb)
            null = C.cast(None, abi.JAC_CB)
            check(ctx.handle, L.b200_problem_set_jac(self._h, null if sparse_proto else self._jac_cb, self._jac_cb if sparse_proto else null))
        self._fin = ctx._adopt(weakref.finalize(self, L.b200_problem_destroy, self._h))

    @property
    def handle(self):
        return self._h

    def set_AB(self, A, B):
        check(self.ctx.handle, lib().b200_problem_set_AB(self._h, float(A), float(B)))

    # plugin-point level access (b1): f!(du,u,p), jvp!(Jv,v,u,p), vjp!
    def residual(self, u, du=None):
        du = du or self.ctx.empty(self.n)
        check(self.ctx.handle, lib().b200_residual(self._h, u.ptr, du.ptr))
        return du

    def jvp(self, u, v, out=None, fd=False):
        out = out or self.ctx.empty(self.n)
        fn = lib().b200_jvp_fd if fd else lib().b200_jvp
        check(self.ctx.handle, fn(self._h, u.ptr, v.ptr, out.ptr))
        return out

    def vjp(self, u, w, out=None):
        out = out or self.ctx.empty(self.n)
        check(self.ctx.handle, lib().b200_vjp(self._h, u.ptr, w.ptr, out.ptr))
        return out

    def residual_jvp(self, u, v):
        du, Jv = self.ctx.empty(self.n), self.ctx.empty(self.n)
        check(self.ctx.handle, lib().b200_residual_jvp(self._h, u.ptr, v.ptr, du.ptr, Jv.ptr))
        return du, Jv

    def residual_norminf(self, u, du=None):
        """(f(u), maximum(abs, f(u))) through the residual kernel's fused norm epilogue (non-finite entries give +inf)."""
        du = du or self.ctx.empty(self.n)
        out = C.c_double()
        check(self.ctx.handle, lib().b200_residual_norminf(self._h, u.ptr, du.ptr, C.byref(out)))
        return du, out.value

    def stencil_plan(self, op):
        """(ring_slots, grid, max_marches) of a Brusselator op (abi.STENCIL_*) on this context; ring_slots == 0: plain kernel."""
        r, g, m = C.c_int32(), C.c_int32(), C.c_int32()
        check(self.ctx.handle, lib().b200_problem_stencil_plan(self._h, int(op), C.byref(r), C.byref(g), C.byref(m)))
        return r.value, g.value, m.value

    def u0(self, mode=abi.U0_REFERENCE):
        u = self.ctx.empty(self.n)
        check(self.ctx.handle, lib().b200_problem_u0(self._h, mode, u.ptr))
        return u

    # dense / sparse Jacobian plumbing (b3)
    def dense_jacobian(self, u):
        J = self.ctx.empty(self.n * self.n)
        check(self.ctx.handle, lib().b200_dense_jac_fill(self._h, u.ptr, J.ptr, self.n))
        return J

    def pattern(self, index_base=1):
        nnz = C.c_int64()
        check(self.ctx.handle, lib().b200_pattern_nnz(self._h, C.byref(nnz)))
        colptr = np.empty(self.n + 1, dtype=np.int64)
        rowval = np.empty(nnz.value, dtype=np.int64)
        check(self.ctx.handle, lib().b200_pattern(self._h, index_base, colptr.ctypes.data_as(C.c_void_p), rowval.ctypes.data_as(C.c_void_p)))
        return colptr, rowval


def coloring_column(n, colptr, rowval, index_base=1, order=abi.ORDER_LARGEST_FIRST):
    """GreedyColoringAlgorithm(LargestFirst()) column colouring (host set-up; bit-exact vs the oracle)."""
    colors = np.empty(n, dtype=np.int64)
    nc = C.c_int64()
    st = lib().b200_coloring_column(n, colptr.ctypes.data_as(C.c_void_p), rowval.ctypes.data_as(C.c_void_p), index_base, order,
                                    colors.ctypes.data_as(C.c_void_p), C.byref(nc))
    if st != abi.OK:
        raise abi.B200Error(st, "b200_coloring_column failed")
    return colors, nc.value


class SparseJacobian:
    """Pattern + colouring + compressed evaluation handle (b200_sparse_jac)."""

    def __init__(self, dprob, colptr=None, rowval=None, colors=None, index_base=1):
        self.dprob, self.ctx = dprob, dprob.ctx
        if colptr is None:
            colptr, rowval = dprob.pattern(index_base)
        if colors is None:
            colors, ncolors = coloring_column(dprob.n, colptr, rowval, index_base)
        else:
            colors = np.ascontiguousarray(colors, dtype=np.int64)
            ncolors = int(colors.max())
        self.colptr, self.rowval, self.colors, self.ncolors, self.index_base = colptr, rowval, colors, ncolors, index_base
        self.nnz = len(rowval)
        self._h = C.c_void_p()
        check(self.ctx.handle, lib().b200_sparse_jac_create(dprob.handle, colptr.ctypes.data_as(C.c_void_p), rowval.ctypes.data_as(C.c_void_p),
                                                            index_base, colors.ctypes.data_as(C.c_void_p), ncolors, C.byref(self._h)))
        self._fin = self.ctx._adopt(weakref.finalize(self, lib().b200_sparse_jac_destroy, self._h))

    def fill(self, u, nzval=None):
        nzval = nzval or self.ctx.empty(self.nnz)
        check(self.ctx.handle, lib().b200_sparse_jac_fill(self._h, u.ptr, nzval.ptr))
        return nzval

    def mul(self, nzval, x, transpose=False):
        y = self.ctx.empty(self.dprob.n)
        fn = lib().b200_spmv_t if transpose else lib().b200_spmv
        check(self.ctx.handle, fn(self._h, nzval.ptr, x.ptr, y.ptr))
        return y


class JacobianOperator:
    """StatefulJacobianOperator(JacobianOperator(prob, fu, u), u, p): matrix-free J(u) with mul! (SciMLJacobianOperators.jl:210-243)."""

    def __init__(self, dprob, u, jvp_autodiff=None):
        self.dprob, self.u = dprob, u
        self.fd = isinstance(jvp_autodiff, AutoFiniteDiff)

    def mul(self, v, out=None):  # mul!(Jv, J, v)
        return self.dprob.jvp(self.u, v, out, fd=self.fd)

    def __matmul__(self, v):
        return self.mul(v)

    def tmul(self, w, out=None):  # mul!(Jtw, transpose(J), w)
        return self.dprob.vjp(self.u, w, out)


class GmresSolver:
    """A LinearSolve-style cache: init once, solve many times (linear_solve.jl:74-147)."""

    def __init__(self, ctx, n, linsolve=None, atol=0.0, rtol=1e-8, keep_hessenberg=0):
        self.ctx, self.n = ctx, n
        g = abi.GmresOpts()
        lib().b200_gmres_opts_default(C.byref(g))
        (linsolve or KrylovJL_GMRES()).fill(g)
        g.atol, g.rtol = float(atol), float(rtol)
        self._h = C.c_void_p()
        check(ctx.handle, lib().b200_gmres_create(ctx.handle, n, C.byref(g), C.byref(self._h)))
        self._fin = ctx._adopt(weakref.finalize(self, lib().b200_gmres_destroy, self._h))
        self.keep = keep_hessenberg
        if keep_hessenberg:
            check(ctx.handle, lib().b200_gmres_keep_hessenberg(self._h, keep_hessenberg))

    def update_tolerances(self, atol=-1.0, rtol=-1.0):
        check(self.ctx.handle, lib().b200_gmres_set_tolerances(self._h, atol, rtol))

    def _op(self, A):
        op = C.c_void_p()
        L = lib()
        keep = None
        if isinstance(A, JacobianOperator):
            check(self.ctx.handle, L.b200_linop_from_problem(A.dprob.handle, A.u.ptr, abi.JVP_FINITE_DIFF if A.fd else abi.JVP_EXACT, C.byref(op)))
        elif isinstance(A, tuple) and A[0] == "csc":
            _, colptr, rowval, nzval, base = A
            check(self.ctx.handle, L.b200_linop_from_csc(self.ctx.handle, self.n, colptr.ptr, rowval.ptr, nzval.ptr, base, C.byref(op)))
        elif isinstance(A, tuple) and A[0] == "dense":
            check(self.ctx.handle, L.b200_linop_from_dense(self.ctx.handle, self.n, A[1].ptr, self.n, C.byref(op)))
        elif isinstance(A, tuple) and A[0] == "sparse_jac":
            check(self.ctx.handle, L.b200_sparse_jac_linop(A[1]._h, A[2].ptr, C.byref(op)))
        elif callable(A):
            n, ctx = self.n, self.ctx

            def mv(user, x, y):
                try:
                    A(DeviceVector(ctx, n, ptr=y), DeviceVector(ctx, n, ptr=x))
                    return 0
                except Exception:  # noqa: BLE001
                    import traceback
                    traceback.print_exc()
                    return 1
            keep = abi.MATVEC_CB(mv)
            check(self.ctx.handle, L.b200_linop_from_callback(self.ctx.handle, self.n, keep, None, C.byref(op)))
        else:
            raise TypeError("unsupported operator")
        return op, keep

    def solve(self, A, b, x=None, Pl=None, Pr=None):
        """Pl / Pr: operator handles that apply the inverse of the left / right preconditioner (e.g. BlockJacobi().linop)."""
        x = x or self.ctx.zeros(self.n)
        op, keep = self._op(A)
        st = abi.GmresStats()
        try:
            check(self.ctx.handle, lib().b200_gmres_set_precond(self._h, Pl, Pr))
            check(self.ctx.handle, lib().b200_gmres_solve(self._h, op, b.ptr, x.ptr, C.byref(st)))
        finally:
            lib().b200_gmres_set_precond(self._h, None, None)
            lib().b200_linop_destroy(op)
            for q in (Pl, Pr):
                if q is not None:
                    lib().b200_linop_destroy(q)
        return x, st

    def hessenberg(self, iters):
        cnt = iters * (iters + 3) // 2
        out = np.empty(cnt)
        check(self.ctx.handle, lib().b200_gmres_get_hessenberg(self._h, out.ctypes.data_as(C.c_void_p), cnt))
        return out


# ----------------------------------------------------------------------------- init / step! / solve! / reinit! / solve
class NonlinearSolveCache:
    """What `init(prob, alg; kwargs...)` returns: persistent device workspace, iterator interface."""

    def __init__(self, prob, alg, abstol=None, reltol=None, maxiters=1000, termination_condition=None, store_trace=True, ctx=None, maxtime=None):
        self.prob, self.alg = prob, alg
        self.ctx = ctx or prob.ctx or default_context()
        self.dprob = _DeviceProblem(self.ctx, prob)
        self.opts = _build_opts(prob, alg, abstol, reltol, maxiters, termination_condition, store_trace, maxtime)
        self._h = C.c_void_p()
        check(self.ctx.handle, lib().b200_newton_create(self.dprob.handle, C.byref(self.opts), C.byref(self._h)))
        self._fin = self.ctx._adopt(weakref.finalize(self, lib().b200_newton_destroy, self._h))
        self.n = self.dprob.n
        self._host_u0 = not isinstance(prob.u0, DeviceVector)
        self.reinit(prob.u0)

    def reinit(self, u0, p=None):  # reinit!(cache, u0; p)
        if p is not None and self.prob.f.builtin and self.prob.f.f.kind in (abi.PROB_BRUSS2D, abi.PROB_BRUSS3D):
            self.dprob.set_AB(p[0], p[1])
        d = _as_device(self.ctx, u0)
        assert d.n == self.n, "u0 has %d entries, problem has %d" % (d.n, self.n)
        check(self.ctx.handle, lib().b200_newton_reinit(self._h, d.ptr))
        self.ctx.sync()
        return self

    def step(self):  # step!(cache)
        t = C.c_int32()
        check(self.ctx.handle, lib().b200_newton_step(self._h, C.byref(t)))
        return bool(t.value)

    def _result(self):
        r = abi.NewtonResult()
        check(self.ctx.handle, lib().b200_newton_result_get(self._h, C.byref(r)))
        return r

    @property
    def u(self):
        p = C.c_void_p()
        check(self.ctx.handle, lib().b200_newton_u(self._h, C.byref(p)))
        return DeviceVector(self.ctx, self.n, ptr=p, owner=self)

    @property
    def fu(self):
        p = C.c_void_p()
        check(self.ctx.handle, lib().b200_newton_fu(self._h, C.byref(p)))
        return DeviceVector(self.ctx, self.n, ptr=p, owner=self)

    def trace(self):
        r = self._result()
        recs = (abi.TraceRec * max(r.ntrace, 1))()
        cnt = C.c_int32()
        check(self.ctx.handle, lib().b200_newton_trace(self._h, recs, r.ntrace, C.byref(cnt)))
        return [recs[i] for i in range(cnt.value)]

    def _solution(self, r, u, resid):
        stats = NLStats(r.nf, r.njacs, r.nfactors, r.nsolve, r.nsteps, r.njvp)
        return NonlinearSolution(self.prob, self.alg, u, resid, r.retcode, stats, self.trace() if self.opts.store_trace else None,
                                 r.bytes, r.resid_inf)

    def solve(self, to_host=None):  # solve!(cache)
        r = abi.NewtonResult()
        check(self.ctx.handle, lib().b200_newton_solve(self._h, C.byref(r)))
        to_host = self._host_u0 if to_host is None else to_host
        u, fu = self.u, self.fu
        if to_host:
            u, fu = u.to_host(), fu.to_host()
        return self._solution(r, u, fu)

    def solve_host(self, u0_host, u_out=None, resid_out=None):
        """The end-to-end call with HOST buffers (H2D of u0, solve, D2H of u and resid) — bench.py's e2e leg."""
        u0_host = np.ascontiguousarray(u0_host, dtype=np.float64)
        u_out = np.empty(self.n) if u_out is None else u_out
        resid_out = np.empty(self.n) if resid_out is None else resid_out
        r = abi.NewtonResult()
        check(self.ctx.handle, lib().b200_newton_solve_host(self._h, u0_host.ctypes.data_as(C.c_void_p), u_out.ctypes.data_as(C.c_void_p),
                                                            resid_out.ctypes.data_as(C.c_void_p), C.byref(r)))
        return self._solution(r, u_out, resid_out)


def init(prob, alg=None, **kw):
    return NonlinearSolveCache(prob, alg or NewtonRaphson(), **kw)


def step_b(cache):
    """step!(cache)"""
    return cache.step()


def solve_b(cache):
    """solve!(cache)"""
    return cache.solve()


def reinit_b(cache, u0, p=None):
    """reinit!(cache, u0; p)"""
    return cache.reinit(u0, p)


# ----------------------------------------------------------------------------- ensemble
class EnsembleProblem:
    """EnsembleProblem(prob; prob_func = (prob, i, repeat) -> remake(prob; ...))."""

    def __init__(self, prob, prob_func=None):
        self.prob, self.prob_func = prob, prob_func


class EnsembleB200:
    """The EnsembleAlgorithm that shards trajectories over ranks (one process per GPU) and batches them per GPU."""

    def __init__(self, rank=0, world_size=1):
        self.rank, self.world_size = rank, world_size


class EnsembleSolution:
    def __init__(self, u, resid_inf, retcodes, nsteps, njvp, summary, lo, hi):
        self.u, self.resid_inf, self.retcodes, self.nsteps, self.njvp, self.summary = u, resid_inf, retcodes, nsteps, njvp, summary
        self.lo, self.hi = lo, hi

    def __len__(self):
        return len(self.retcodes)

    def converged(self):
        return bool(np.all(self.retcodes == ReturnCode.Success))


def shard_range(K, rank, world_size):
    """Contiguous trajectory block of `rank` (SURVEY.md §8e): [lo, hi)."""
    base, rem = divmod(K, world_size)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


class EnsembleCache:
    """Persistent per-GPU batch workspace for K_local 2D-Brusselator trajectories.  The options are those of a single solve,
    preconditioner included (`Multigrid` on either side is batched, `BlockJacobi` runs trajectory by trajectory; ILU0 and the
    AMGs need an assembled Jacobian and are refused).  `alg` is `NewtonRaphson(linsolve = KrylovJL_GMRES(...))`, with or
    without `linesearch = BackTracking()`, or `TrustRegion(linsolve = KrylovJL_GMRES(...))`; the globalised ones take no
    preconditioner (refused otherwise), and the Bastin radius scheme runs trajectory by trajectory.  Option sets the batched
    kernel does not implement (see csrc/ens_batched.cu) run each trajectory through the general driver."""

    def __init__(self, ctx, N, nprob_local, alpha, alg, abstol=None, reltol=None, maxiters=1000, termination_condition=None, maxtime=None):
        self.ctx, self.N, self.K, self.n = ctx, N, nprob_local, 2 * N * N
        dummy = NonlinearProblem(Brusselator2D(N), None, (3.4, 1.0, alpha))
        self.opts = _build_opts(dummy, alg, abstol, reltol, maxiters, termination_condition, False, maxtime)
        self._h = C.c_void_p()
        check(ctx.handle, lib().b200_ens_create(ctx.handle, N, nprob_local, float(alpha), C.byref(self.opts), C.byref(self._h)))
        self._fin = ctx._adopt(weakref.finalize(self, lib().b200_ens_destroy, self._h))
        self.u_out = ctx.empty(self.K * self.n)
        self.resid = ctx.empty(self.K)
        self.rc = ctx.empty(self.K, np.int32)
        self.ns = ctx.empty(self.K, np.int32)
        self.nj = ctx.empty(self.K, np.int32)

    def solve(self, u0_dev, A_dev, B_dev):
        res = abi.EnsResult()
        check(self.ctx.handle, lib().b200_ens_solve(self._h, u0_dev.ptr, A_dev.ptr, B_dev.ptr, self.u_out.ptr, self.resid.ptr, self.rc.ptr,
                                                    self.ns.ptr, self.nj.ptr, C.byref(res)))
        return res

    def precond_apply(self, u_dev, A_dev, x_dev, y_dev=None):
        """y_m = M_m^-1 x_m for every trajectory of a batched multigrid ensemble, M_m the V-cycle at iterate u_m with parameter
        A_m, by the solve kernel's own routine (u, x, y: K x n device vectors, A: K).  Returns y."""
        y_dev = self.ctx.empty(self.K * self.n) if y_dev is None else y_dev
        check(self.ctx.handle, lib().b200_ens_precond_apply(self._h, u_dev.ptr, A_dev.ptr, x_dev.ptr, y_dev.ptr))
        return y_dev

    def ctas_per_sm(self):
        """Resident CTAs per SM of the batched solve kernel for these options (0 when trajectories take the general driver)."""
        v = C.c_int32()
        check(self.ctx.handle, lib().b200_ens_ctas_per_sm(self._h, C.byref(v)))
        return v.value


class Communicator:
    """The collective step of the ensemble path through the library's own C-ABI entry points (b200_nccl_init /
    b200_ens_allgather / b200_ens_allreduce_stats): NCCL over NVLink, enqueued on the context's stream.  One process per GPU:
    rank 0 calls `Communicator.unique_id()` and ships the 128 bytes to the other ranks (any host-side channel)."""

    @staticmethod
    def unique_id():
        buf = (C.c_ubyte * 128)()
        st = lib().b200_nccl_unique_id(buf)
        if st != 0:
            raise abi.B200Error(st, "b200_nccl_unique_id failed (libnccl.so.2 not loadable?)")
        return bytes(buf)

    @staticmethod
    def nccl_version():
        v = C.c_int32(0)
        return v.value if lib().b200_nccl_version(C.byref(v)) == 0 else None

    def __init__(self, ctx, nranks, rank, unique_id):
        self.ctx, self.nranks, self.rank = ctx, nranks, rank
        self._h = C.c_void_p()
        buf = (C.c_ubyte * 128).from_buffer_copy(unique_id)
        check(ctx.handle, lib().b200_nccl_init(ctx.handle, nranks, rank, buf, C.byref(self._h)))
        self._fin = ctx._adopt(weakref.finalize(self, lib().b200_nccl_destroy, self._h))

    def allgather(self, u_local, u_all):
        check(self.ctx.handle, lib().b200_ens_allgather(self._h, u_local.ptr, u_local.n, u_all.ptr))

    def allreduce_stats(self, local):
        out = abi.EnsResult()
        check(self.ctx.handle, lib().b200_ens_allreduce_stats(self._h, C.byref(local), C.byref(out)))
        return out

    def allreduce_stats_begin(self, local):
        check(self.ctx.handle, lib().b200_ens_allreduce_stats_begin(self._h, C.byref(local)))

    def allreduce_stats_finish(self):
        out = abi.EnsResult()
        check(self.ctx.handle, lib().b200_ens_allreduce_stats_finish(self._h, C.byref(out)))
        return out


def _solve_ensemble(ens, alg, ensalg, trajectories, ctx=None, **kw):
    prob = ens.prob
    assert prob.f.builtin and prob.f.f.kind == abi.PROB_BRUSS2D, "EnsembleB200 batches 2D Brusselator trajectories"
    ctx = ctx or prob.ctx or default_context()
    N = prob.f.f.N
    n = 2 * N * N
    lo, hi = shard_range(trajectories, ensalg.rank, ensalg.world_size)
    K = hi - lo
    u0 = np.empty((K, n))
    A = np.empty(K)
    B = np.empty(K)
    alpha = None
    for m in range(lo, hi):  # prob_func(prob, i, repeat), 1-based i as in Julia
        pm = ens.prob_func(prob, m + 1, 1) if ens.prob_func else prob
        u0[m - lo] = np.asarray(pm.u0, dtype=np.float64).ravel(order="F")
        A[m - lo], B[m - lo] = pm.p[0], pm.p[1]
        alpha = pm.p[2] if alpha is None else alpha
        assert pm.p[2] == alpha, "alpha must be shared by all trajectories of a batch"
    cache = EnsembleCache(ctx, N, K, alpha, alg, **kw)
    res = cache.solve(ctx.to_device(u0.ravel()), ctx.to_device(A), ctx.to_device(B))
    return EnsembleSolution(cache.u_out.to_host().reshape(K, n), cache.resid.to_host(), cache.rc.to_host(), cache.ns.to_host(),
                            cache.nj.to_host(), res, lo, hi)


def solve(prob, alg=None, ensemblealg=None, trajectories=None, **kw):
    """solve(prob, alg; abstol, reltol, maxiters, termination_condition, store_trace)  /  solve(ensembleprob, alg, EnsembleB200(); trajectories)."""
    if isinstance(prob, EnsembleProblem):
        return _solve_ensemble(prob, alg or NewtonRaphson(linsolve=KrylovJL_GMRES()), ensemblealg or EnsembleB200(), trajectories, **kw)
    return init(prob, alg, **kw).solve()
