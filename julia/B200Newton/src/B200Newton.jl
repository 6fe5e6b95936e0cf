# B200Newton.jl — thin Julia glue over libb200newton.so (include/b200newton.h).  `@ccall` only: no CUDA.jl, no
# KernelAbstractions, no CPU fallback.  It plugs the library into NonlinearSolve.jl's own extension points:
#
#   b1  NonlinearFunction{true}(f!; jvp = jvp!)                 -> `brusselator_function(prob)` returns callable structs
#   b4  linsolve = B200GMRES()  (a LinearSolve.SciMLLinearSolveAlgorithm, needs_concrete_A = false)
#   b5  B200Vector <: AbstractVector{Float64}                    (device array the generic layers can carry around)
#   b6  EnsembleB200 <: SciMLBase.EnsembleAlgorithm              (gather through the library's own NCCL entry points)
#   +   B200NewtonKrylov <: AbstractNonlinearSolveAlgorithm      whole-solve fast path (pattern: ext/NonlinearSolvePETScExt.jl:38-167)
#
# NOTE: this file cannot be executed in the build environment (no Julia runtime, SURVEY.md §0).  It is kept mechanical — one
# `@ccall` per exported symbol — and is checked statically (tests/test_julia_glue_layout.py: struct layouts, every `@ccall`
# signature against the header, no positional construction of the option structs).  The same call sequences are executed
# on the GPU by the Python harness (nonlinearsolve.jl_b200/api.py) and by the plain-C host tests/abi_c/abi_c_check.c.
module B200Newton

using LinearAlgebra
using SparseArrays: SparseMatrixCSC
import SciMLBase
import SciMLBase: ReturnCode, NLStats
import CommonSolve
import LinearSolve
import NonlinearSolveBase
import SciMLJacobianOperators
import ArrayInterface

const libb200 = get(ENV, "B200NEWTON_LIB", joinpath(@__DIR__, "..", "..", "..", "nonlinearsolve.jl_b200", "libb200newton.so"))

# ------------------------------------------------------------------ status handling
struct B200Error <: Exception
    code::Int32
    msg::String
end
const Ctx = Ptr{Cvoid}

function check(ctx::Ctx, status::Int32)
    status == 0 && return nothing
    msg = ctx == C_NULL ? "" : unsafe_string(@ccall libb200.b200_last_error(ctx::Ctx)::Cstring)
    throw(B200Error(status, msg))
end

# SciMLBase.ReturnCode <- B200_RC_* (include/b200newton.h)
const RETCODES = (ReturnCode.Default, ReturnCode.Success, ReturnCode.MaxIters, ReturnCode.MaxTime, ReturnCode.Stalled,
    ReturnCode.StalledSuccess, ReturnCode.Unstable, ReturnCode.InternalLinearSolveFailed,
    ReturnCode.InternalLineSearchFailed, ReturnCode.ShrinkThresholdExceeded, ReturnCode.InitialFailure, ReturnCode.Failure,
    ReturnCode.ConvergenceFailure)
retcode(c::Integer) = RETCODES[c + 1]

# ------------------------------------------------------------------ context (one per task per device)
mutable struct Context
    handle::Ctx
    device::Int
    function Context(device::Integer = 0)
        h = Ref{Ctx}(C_NULL)
        st = @ccall libb200.b200_ctx_create(device::Int32, C_NULL::Ptr{Cvoid}, h::Ref{Ctx})::Int32
        st == -6 && throw(B200Error(st, "no CUDA device: the B200 backend has no CPU fallback"))
        check(C_NULL, st)
        ctx = new(h[], device)
        finalizer(c -> (@ccall libb200.b200_ctx_destroy(c.handle::Ctx)::Int32), ctx)
        return ctx
    end
end
const DEFAULT_CTX = Dict{Int, Context}()
default_context(device::Integer = 0) = get!(() -> Context(device), DEFAULT_CTX, Int(device))
sync(ctx::Context) = check(ctx.handle, @ccall libb200.b200_ctx_sync(ctx.handle::Ctx)::Int32)
function device_count()
    n = Ref{Int32}(0)
    @ccall libb200.b200_device_count(n::Ref{Int32})::Int32
    return Int(n[])
end

# ------------------------------------------------------------------ raw device buffers (Int32 / Float64 result arrays)
mutable struct DeviceBuffer{T}
    ctx::Context
    ptr::Ptr{T}
    n::Int
    function DeviceBuffer{T}(ctx::Context, n::Integer) where {T}
        p = Ref{Ptr{Cvoid}}(C_NULL)
        check(ctx.handle, @ccall libb200.b200_malloc(ctx.handle::Ctx, (sizeof(T) * n)::Csize_t, p::Ref{Ptr{Cvoid}})::Int32)
        b = new{T}(ctx, Ptr{T}(p[]), n)
        finalizer(x -> (@ccall libb200.b200_free(x.ctx.handle::Ctx, x.ptr::Ptr{Cvoid})::Int32), b)
        return b
    end
end
function Base.Array(b::DeviceBuffer{T}) where {T}
    out = Vector{T}(undef, b.n)
    GC.@preserve out check(b.ctx.handle, @ccall libb200.b200_memcpy_d2h(b.ctx.handle::Ctx, pointer(out)::Ptr{Cvoid}, b.ptr::Ptr{Cvoid}, (sizeof(T) * b.n)::Csize_t)::Int32)
    return out
end

# ------------------------------------------------------------------ b5: device vector
# `owner` keeps the allocation alive for views (vec / reshape of the same memory, library-owned buffers wrapped in place).
mutable struct B200Vector <: AbstractVector{Float64}
    ctx::Context
    ptr::Ptr{Float64}
    n::Int
    owner::Any
    function B200Vector(ctx::Context, n::Integer)
        p = Ref{Ptr{Cvoid}}(C_NULL)
        check(ctx.handle, @ccall libb200.b200_malloc(ctx.handle::Ctx, (8 * n)::Csize_t, p::Ref{Ptr{Cvoid}})::Int32)
        v = new(ctx, Ptr{Float64}(p[]), n, nothing)
        finalizer(x -> (@ccall libb200.b200_free(x.ctx.handle::Ctx, x.ptr::Ptr{Cvoid})::Int32), v)
        return v
    end
    # non-owning view of device memory that `owner` (another vector, a solver cache, the library) keeps alive
    B200Vector(ctx::Context, ptr::Ptr{Float64}, n::Integer, owner) = new(ctx, ptr, n, owner)
end
unsafe_wrap_device(ctx::Context, p::Ptr{Float64}, n::Integer, owner = nothing) = B200Vector(ctx, p, n, owner)

Base.size(v::B200Vector) = (v.n,)
Base.length(v::B200Vector) = v.n
Base.eltype(::Type{B200Vector}) = Float64
Base.IndexStyle(::Type{B200Vector}) = IndexLinear()
Base.similar(v::B200Vector) = B200Vector(v.ctx, v.n)
Base.similar(v::B200Vector, ::Type{Float64}) = B200Vector(v.ctx, v.n)
Base.similar(v::B200Vector, ::Type{Float64}, dims::Tuple{Int}) = B200Vector(v.ctx, dims[1])
Base.zero(v::B200Vector) = fill!(similar(v), 0.0)
Base.vec(v::B200Vector) = v
Base.reshape(v::B200Vector, dims::Tuple{Int}) = (dims[1] == v.n || throw(DimensionMismatch()); v)
Base.reshape(v::B200Vector, ::Colon) = v
# the generic layers never index a device array: ArrayInterface.fast_scalar_indexing(::B200Vector) == false routes them
# to the mapreduce / broadcast forms below (utils.jl:17, 45-58, 81-96; common_defaults.jl:19-37)
Base.getindex(::B200Vector, ::Int) = error("scalar indexing of a B200Vector is disabled (ArrayInterface.fast_scalar_indexing == false)")
Base.setindex!(::B200Vector, _, ::Int) = error("scalar indexing of a B200Vector is disabled (ArrayInterface.fast_scalar_indexing == false)")
ArrayInterface.fast_scalar_indexing(::Type{B200Vector}) = false
ArrayInterface.can_setindex(::Type{B200Vector}) = true      # `fill!`, `copyto!` and in-place broadcast are provided
ArrayInterface.device(::Type{B200Vector}) = ArrayInterface.GPU()

function B200Vector(ctx::Context, x::AbstractArray{<:Real})
    v = B200Vector(ctx, length(x))
    copyto!(v, vec(collect(Float64, x)))
end
function Base.copyto!(dst::B200Vector, src::Array{Float64})
    length(src) == dst.n || throw(DimensionMismatch())
    GC.@preserve src check(dst.ctx.handle, @ccall libb200.b200_memcpy_h2d(dst.ctx.handle::Ctx, dst.ptr::Ptr{Cvoid}, pointer(src)::Ptr{Cvoid}, (8 * dst.n)::Csize_t)::Int32)
    return dst
end
function Base.copyto!(dst::Array{Float64}, src::B200Vector)
    length(dst) == src.n || throw(DimensionMismatch())
    GC.@preserve dst check(src.ctx.handle, @ccall libb200.b200_memcpy_d2h(src.ctx.handle::Ctx, pointer(dst)::Ptr{Cvoid}, src.ptr::Ptr{Cvoid}, (8 * src.n)::Csize_t)::Int32)
    return dst
end
function Base.copyto!(dst::B200Vector, src::B200Vector)
    dst.ptr == src.ptr && return dst
    check(dst.ctx.handle, @ccall libb200.b200_copy(dst.ctx.handle::Ctx, dst.n::Int64, src.ptr::Ptr{Float64}, dst.ptr::Ptr{Float64})::Int32)
    return dst
end
Base.Array(v::B200Vector) = copyto!(Vector{Float64}(undef, v.n), v)
Base.collect(v::B200Vector) = Array(v)
Base.copy(v::B200Vector) = copyto!(similar(v), v)
Base.fill!(v::B200Vector, a::Real) = (check(v.ctx.handle, @ccall libb200.b200_fill(v.ctx.handle::Ctx, v.n::Int64, Float64(a)::Float64, v.ptr::Ptr{Float64})::Int32); v)
Base.show(io::IO, v::B200Vector) = print(io, "B200Vector(", v.n, " Float64 on device ", v.ctx.device, ")")
Base.show(io::IO, ::MIME"text/plain", v::B200Vector) = show(io, v)

# ---- the BLAS-1 surface L2-L4 and Krylov.jl touch (SURVEY.md §8b b5)
function LinearAlgebra.axpy!(a::Real, x::B200Vector, y::B200Vector)
    check(y.ctx.handle, @ccall libb200.b200_axpy(y.ctx.handle::Ctx, y.n::Int64, Float64(a)::Float64, x.ptr::Ptr{Float64}, y.ptr::Ptr{Float64})::Int32); y
end
function LinearAlgebra.axpby!(a::Real, x::B200Vector, b::Real, y::B200Vector)
    check(y.ctx.handle, @ccall libb200.b200_axpby(y.ctx.handle::Ctx, y.n::Int64, Float64(a)::Float64, x.ptr::Ptr{Float64}, Float64(b)::Float64, y.ptr::Ptr{Float64})::Int32); y
end
LinearAlgebra.rmul!(x::B200Vector, a::Real) = (check(x.ctx.handle, @ccall libb200.b200_scal(x.ctx.handle::Ctx, x.n::Int64, Float64(a)::Float64, x.ptr::Ptr{Float64})::Int32); x)
LinearAlgebra.lmul!(a::Real, x::B200Vector) = rmul!(x, a)
function LinearAlgebra.dot(x::B200Vector, y::B200Vector)
    r = Ref{Float64}(0.0)
    check(x.ctx.handle, @ccall libb200.b200_dot(x.ctx.handle::Ctx, x.n::Int64, x.ptr::Ptr{Float64}, y.ptr::Ptr{Float64}, r::Ref{Float64})::Int32)
    return r[]
end
function LinearAlgebra.norm(x::B200Vector, p::Real = 2)
    r = Ref{Float64}(0.0)
    if p == 2
        check(x.ctx.handle, @ccall libb200.b200_nrm2(x.ctx.handle::Ctx, x.n::Int64, x.ptr::Ptr{Float64}, r::Ref{Float64})::Int32)
    elseif p == Inf
        check(x.ctx.handle, @ccall libb200.b200_norminf(x.ctx.handle::Ctx, x.n::Int64, x.ptr::Ptr{Float64}, r::Ref{Float64})::Int32)
    else
        error("only the 2- and Inf-norms are provided on the device")
    end
    return r[]
end
function extrema_device(x::B200Vector)
    lo = Ref{Float64}(0.0); hi = Ref{Float64}(0.0)
    check(x.ctx.handle, @ccall libb200.b200_extrema(x.ctx.handle::Ctx, x.n::Int64, x.ptr::Ptr{Float64}, lo::Ref{Float64}, hi::Ref{Float64})::Int32)
    return lo[], hi[]
end
Base.extrema(x::B200Vector) = extrema_device(x)        # trust_region.jl:330-337 (max_trust_radius from the state's range)
Base.maximum(x::B200Vector) = extrema_device(x)[2]
Base.minimum(x::B200Vector) = extrema_device(x)[1]
Base.maximum(::typeof(abs), x::B200Vector) = norm(x, Inf)   # common_defaults.jl:37  Linf_NORM
Base.sum(::typeof(abs2), x::B200Vector) = dot(x, x)
Base.any(::typeof(isnan), x::B200Vector) = isnan(norm(x, Inf))   # the device max-reduction propagates non-finite entries
function Base.:(==)(x::B200Vector, y::B200Vector)            # termination_conditions.jl:446
    x.n == y.n || return false
    r = Ref{Int32}(0)
    check(x.ctx.handle, @ccall libb200.b200_equal(x.ctx.handle::Ctx, x.n::Int64, x.ptr::Ptr{Float64}, y.ptr::Ptr{Float64}, r::Ref{Int32})::Int32)
    return r[] == 1
end
function diffnrm2(x::B200Vector, y::B200Vector)
    r = Ref{Float64}(0.0)
    check(x.ctx.handle, @ccall libb200.b200_diffnrm2(x.ctx.handle::Ctx, x.n::Int64, x.ptr::Ptr{Float64}, y.ptr::Ptr{Float64}, r::Ref{Float64})::Int32)
    return r[]
end
# mapreduce: the one-argument forms the reference calls on a state vector (common_defaults.jl:1-4, :37) ...
Base.mapreduce(::typeof(abs), ::typeof(max), x::B200Vector; kw...) = norm(x, Inf)
Base.mapreduce(::typeof(abs2), ::typeof(+), x::B200Vector; kw...) = dot(x, x)
Base.mapreduce(::typeof(abs2), ::typeof(Base.add_sum), x::B200Vector; kw...) = dot(x, x)
Base.mapreduce(::typeof(NonlinearSolveBase.UNITLESS_ABS2), ::typeof(NonlinearSolveBase.Utils.abs2_and_sum), x::B200Vector; kw...) = dot(x, x)
# ... and the two-argument helpers built on closures (utils.jl:45-58, 80-99), specialised on the helper itself because a
# closure cannot be shipped to the device: ||x - y||, ||x + y|| in the 2- and Inf-norms
function NonlinearSolveBase.Utils.norm_op(::typeof(NonlinearSolveBase.L2_NORM), op::Union{typeof(+), typeof(-)}, x::B200Vector, y::B200Vector)
    op === (-) && return diffnrm2(x, y)
    t = copy(x); axpy!(1.0, y, t)
    return norm(t, 2)
end
function NonlinearSolveBase.Utils.nonallocating_maximum(op::Union{typeof(+), typeof(-)}, x::B200Vector, y::B200Vector)
    t = copy(x); axpy!(op === (-) ? -1.0 : 1.0, y, t)
    return norm(t, Inf)
end

# ---- broadcast: the driver's in-place updates are all linear combinations of device vectors with host scalars
# (`@. δu *= -1` newton.jl:138, `@bb axpy!` solve.jl:438, `@. u_cache = u + δu` trust_region.jl:399, the dogleg blends
# dogleg.jl:117-149) plus the elementwise product.  The broadcast tree is flattened into  sum_i c_i x_i  and evaluated
# with axpby / axpy; any other expression raises an error naming the supported forms (no silent host fallback).
struct B200Style <: Base.Broadcast.AbstractArrayStyle{1} end
B200Style(::Val{1}) = B200Style()
B200Style(::Val{N}) where {N} = Base.Broadcast.DefaultArrayStyle{N}()
Base.BroadcastStyle(::Type{B200Vector}) = B200Style()
Base.BroadcastStyle(::B200Style, ::Base.Broadcast.DefaultArrayStyle{0}) = B200Style()

const Term = Tuple{Float64, B200Vector}
_lin(x::B200Vector) = Term[(1.0, x)]
_lin(x::Base.RefValue) = nothing
_lin(::Any) = nothing
_scalar(x::Real) = Float64(x)
_scalar(x::Base.RefValue{<:Real}) = Float64(x[])
_scalar(x::Base.Broadcast.Broadcasted{<:Any, <:Any, <:Any, <:Tuple{Vararg{Union{Real, Base.RefValue{<:Real}, Base.Broadcast.Broadcasted}}}}) =
    (a = map(_scalar, x.args); any(isnothing, a) ? nothing : Float64(x.f(a...)))   # scalar sub-expression such as (d_cauchy / l_grad)
_scalar(::Any) = nothing
function _lin(bc::Base.Broadcast.Broadcasted)
    f, a = bc.f, bc.args
    if f === (+) || f === (-)
        if length(a) == 1
            t = _lin(a[1]); t === nothing && return nothing
            return f === (-) ? Term[(-c, x) for (c, x) in t] : t
        end
        out = _lin(a[1]); out === nothing && return nothing
        for q in a[2:end]
            t = _lin(q); t === nothing && return nothing
            append!(out, f === (-) ? Term[(-c, x) for (c, x) in t] : t)
        end
        return out
    elseif f === (*)
        vecs = [q for q in a if _scalar(q) === nothing]
        length(vecs) == 1 || return nothing                     # at most one vector factor (x .* y is handled separately)
        s = prod(Float64[_scalar(q) for q in a if _scalar(q) !== nothing]; init = 1.0)
        t = _lin(vecs[1]); t === nothing && return nothing
        return Term[(s * c, x) for (c, x) in t]
    elseif f === (/) && length(a) == 2 && _scalar(a[2]) !== nothing
        t = _lin(a[1]); t === nothing && return nothing
        return Term[(c / _scalar(a[2]), x) for (c, x) in t]
    elseif f === identity && length(a) == 1
        return _lin(a[1])
    end
    return nothing
end
function Base.copyto!(dest::B200Vector, bc::Base.Broadcast.Broadcasted{B200Style})
    if bc.f === (*) && length(bc.args) == 2 && bc.args[1] isa B200Vector && bc.args[2] isa B200Vector   # z = x .* y
        x, y = bc.args
        check(dest.ctx.handle, @ccall libb200.b200_mul(dest.ctx.handle::Ctx, dest.n::Int64, x.ptr::Ptr{Float64}, y.ptr::Ptr{Float64}, dest.ptr::Ptr{Float64})::Int32)
        return dest
    end
    if (s = _scalar(bc)) !== nothing
        return fill!(dest, s)
    end
    terms = _lin(bc)
    terms === nothing && error("B200Vector broadcast supports linear combinations of device vectors with host scalars " *
                               "(a .* x .+ b .* y .- z, x ./ a, -x) and x .* y; got " * string(bc.f))
    # the destination may appear on the right-hand side: fold its coefficient into the scaling of dest
    cself = sum(Float64[c for (c, x) in terms if x.ptr == dest.ptr]; init = 0.0)
    others = Term[(c, x) for (c, x) in terms if x.ptr != dest.ptr]
    if isempty(others)
        rmul!(dest, cself)
    else
        axpby!(others[1][1], others[1][2], cself, dest)
        for (c, x) in others[2:end]
            axpy!(c, x, dest)
        end
    end
    return dest
end
Base.copyto!(dest::B200Vector, bc::Base.Broadcast.Broadcasted{<:Base.Broadcast.AbstractArrayStyle{0}}) = fill!(dest, Float64(bc[]))
Base.similar(bc::Base.Broadcast.Broadcasted{B200Style}, ::Type{Float64}) = similar(_first_vector(bc))
_first_vector(x::B200Vector) = x
_first_vector(::Any) = nothing
function _first_vector(bc::Base.Broadcast.Broadcasted)
    for a in bc.args
        v = _first_vector(a)
        v === nothing || return v
    end
    return nothing
end

# ------------------------------------------------------------------ b1: built-in device problems as f! / jvp! / vjp!
mutable struct Problem
    ctx::Context
    handle::Ptr{Cvoid}
    n::Int
    N::Int
    dim::Int
end
function brusselator(ctx::Context, dim::Integer, N::Integer, A, B, alpha)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    if dim == 2
        check(ctx.handle, @ccall libb200.b200_problem_create_bruss2d(ctx.handle::Ctx, N::Int32, Float64(A)::Float64, Float64(B)::Float64, Float64(alpha)::Float64, h::Ref{Ptr{Cvoid}})::Int32)
    else
        check(ctx.handle, @ccall libb200.b200_problem_create_bruss3d(ctx.handle::Ctx, N::Int32, Float64(A)::Float64, Float64(B)::Float64, Float64(alpha)::Float64, h::Ref{Ptr{Cvoid}})::Int32)
    end
    p = Problem(ctx, h[], 2 * N^dim, N, dim)
    finalizer(x -> (@ccall libb200.b200_problem_destroy(x.handle::Ptr{Cvoid})::Int32), p)
    return p
end
"""reference initial condition (sparsity_tests__item1.jl:38-50); `perturbed = true`: the z-perturbed 3D variant of SURVEY.md §8d"""
function initial_condition(prob::Problem; perturbed::Bool = false)
    u = B200Vector(prob.ctx, prob.n)
    check(prob.ctx.handle, @ccall libb200.b200_problem_u0(prob.handle::Ptr{Cvoid}, (perturbed ? 1 : 0)::Int32, u.ptr::Ptr{Float64})::Int32)
    return u
end
residual!(du::B200Vector, u::B200Vector, prob::Problem) = (check(prob.ctx.handle, @ccall libb200.b200_residual(prob.handle::Ptr{Cvoid}, u.ptr::Ptr{Float64}, du.ptr::Ptr{Float64})::Int32); nothing)
jvp!(Jv::B200Vector, v::B200Vector, u::B200Vector, prob::Problem) = (check(prob.ctx.handle, @ccall libb200.b200_jvp(prob.handle::Ptr{Cvoid}, u.ptr::Ptr{Float64}, v.ptr::Ptr{Float64}, Jv.ptr::Ptr{Float64})::Int32); nothing)
vjp!(Jtw::B200Vector, w::B200Vector, u::B200Vector, prob::Problem) = (check(prob.ctx.handle, @ccall libb200.b200_vjp(prob.handle::Ptr{Cvoid}, u.ptr::Ptr{Float64}, w.ptr::Ptr{Float64}, Jtw.ptr::Ptr{Float64})::Int32); nothing)

# callable structs instead of closures, so that the linear solver can recognise "this JacobianOperator is one of ours" and
# hand the built-in fused operator to the library (`device_problem` below) instead of calling back per Arnoldi step
struct B200Residual <: Function
    prob::Problem
end
struct B200JVP <: Function
    prob::Problem
end
struct B200VJP <: Function
    prob::Problem
end
(f::B200Residual)(du, u, p) = residual!(vec(du), vec(u), f.prob)
(f::B200JVP)(Jv, v, u, p) = jvp!(vec(Jv), vec(v), vec(u), f.prob)          # arrays arrive as reshaped views (SciMLJacobianOperators.jl:410)
(f::B200VJP)(Jtw, w, u, p) = vjp!(vec(Jtw), vec(w), vec(u), f.prob)

"""
    brusselator_function(prob) -> NonlinearFunction{true}

`NonlinearFunction{true}(f!; jvp = jvp!, vjp = vjp!)` whose callables run the fused sm_90a kernels (b1).  With it
`solve(NonlinearProblem(fn, u0::B200Vector, p), NewtonRaphson(linsolve = B200GMRES()))` runs the reference's own driver
(`step!`, termination, stats) over device arrays, every arithmetic step in libb200newton.
"""
brusselator_function(prob::Problem) = SciMLBase.NonlinearFunction{true}(B200Residual(prob); jvp = B200JVP(prob), vjp = B200VJP(prob))

# `prepare_jvp` returns a user `f.jvp` verbatim (SciMLJacobianOperators.jl:377), so it sits in `jvp_op`
device_problem(J::SciMLJacobianOperators.JacobianOperator) = J.jvp_op isa B200JVP ? J.jvp_op.prob : nothing
device_problem(J::SciMLJacobianOperators.StatefulJacobianOperator) = device_problem(J.jac_op)
device_problem(::Any) = nothing
linearisation_point(J::SciMLJacobianOperators.StatefulJacobianOperator) = J.u
linearisation_point(::Any) = nothing

# ------------------------------------------------------------------ option structs (bit-compatible with the header)
struct GmresOpts
    memory::Int32; restart::Int32; itmax::Int32; orth::Int32; warm_start::Int32; engine::Int32; check_every::Int32; block::Int32
    atol::Float64; rtol::Float64
end
struct GmresStats
    status::Int32; iters::Int32; nmatvec::Int32; restarts::Int32
    rnorm0::Float64; rnorm::Float64; tol::Float64; bytes::Float64
end
struct NewtonOpts
    abstol::Float64; reltol::Float64
    maxiters::Int32; linsolve::Int32; jvp_mode::Int32; globalization::Int32; forcing::Int32; termination::Int32; store_trace::Int32; fused_step::Int32
    gmres::GmresOpts
    ew_eta0::Float64; ew_eta_max::Float64; ew_gamma::Float64; ew_alpha::Float64; ew_safeguard_threshold::Float64
    ew_safeguard::Int32; max_shrink_times::Int32
    tr_step_threshold::Float64; tr_shrink_threshold::Float64; tr_expand_threshold::Float64; tr_shrink_factor::Float64
    tr_expand_factor::Float64; tr_max_trust_radius::Float64; tr_initial_trust_radius::Float64
    ls_c1::Float64; ls_rho_hi::Float64; ls_rho_lo::Float64; ls_maxiters::Int32; precond::Int32
    descent::Int32; tr_scheme::Int32; pt_alpha_initial::Float64
    maxtime::Float64; term_norm::Int32; term_max_stalled_steps::Int32
    lm_damping_initial::Float64; lm_damping_increase::Float64; lm_damping_decrease::Float64; lm_finite_diff_step::Float64
    lm_alpha_geodesic::Float64; lm_b_uphill::Float64; lm_min_damping_D::Float64; lm_disable_geodesic::Int32; reserved0::Int32
    qn_init_jacobian::Int32; qn_update_rule::Int32; qn_max_resets::Int32; qn_threshold::Int32
    qn_reset_tolerance::Float64; qn_alpha::Float64
end
struct NewtonResult
    retcode::Int32; nsteps::Int32; nf::Int32; njacs::Int32; nfactors::Int32; nsolve::Int32; njvp::Int32; ntrace::Int32
    resid_inf::Float64; bytes::Float64
end
struct EnsResult
    nprob::Int32; nsuccess::Int32; max_nsteps::Int32; reserved::Int32
    total_nsteps::Int64; total_njvp::Int64; worst_resid_inf::Float64
end
"""The option structs are NEVER built positionally: start from the library's defaults and replace fields by name."""
function with(o::T; kw...) where {T <: Union{GmresOpts, NewtonOpts}}
    for k in keys(kw)
        hasfield(T, k) || throw(ArgumentError("$(T) has no field $(k)"))
    end
    vals = ntuple(i -> (nm = fieldname(T, i); haskey(kw, nm) ? convert(fieldtype(T, i), kw[nm]) : getfield(o, i)), fieldcount(T))
    return T(vals...)
end
function default_newton_opts()
    r = Ref{NewtonOpts}()
    @ccall libb200.b200_newton_opts_default(r::Ref{NewtonOpts})::Cvoid
    return r[]
end
function default_gmres_opts()
    r = Ref{GmresOpts}()
    @ccall libb200.b200_gmres_opts_default(r::Ref{GmresOpts})::Cvoid
    return r[]
end
orth_code(s::Symbol) = s === :mgs ? Int32(0) : s === :cgs ? Int32(1) : s === :cgs2 ? Int32(2) : throw(ArgumentError("orth must be :mgs, :cgs or :cgs2"))

# ------------------------------------------------------------------ b4: custom LinearSolve algorithm
"""
    B200GMRES(; restart = 0, memory = 20, orth = :mgs)

`LinearSolve.SciMLLinearSolveAlgorithm` with `needs_concrete_A == false`, so `construct_jacobian_cache` hands it the
matrix-free `JacobianOperator` (jacobian.jl:43-47).  `solve!` runs the device-resident GMRES; when `A` wraps a
`brusselator_function` the operator is the built-in fused kernel (resident Arnoldi engine), otherwise `mul!(w, A, v)` is
called back between kernels.  `orth = :mgs` is Krylov.jl's default (no reorthogonalisation), `:cgs2` reorthogonalises.
"""
Base.@kwdef struct B200GMRES <: LinearSolve.SciMLLinearSolveAlgorithm
    restart::Int = 0
    memory::Int = 20
    orth::Symbol = :mgs
end
LinearSolve.needs_concrete_A(::B200GMRES) = false
LinearSolve.needs_square_A(::B200GMRES) = true

mutable struct GmresCache
    handle::Ptr{Cvoid}
    n::Int
end
function LinearSolve.init_cacheval(alg::B200GMRES, A, b::B200Vector, u, Pl, Pr, maxiters::Int, abstol, reltol, verbose, assumptions)
    o = Ref(with(default_gmres_opts(); memory = alg.memory, restart = alg.restart, itmax = maxiters, orth = orth_code(alg.orth), atol = abstol, rtol = reltol))
    h = Ref{Ptr{Cvoid}}(C_NULL)
    check(b.ctx.handle, @ccall libb200.b200_gmres_create(b.ctx.handle::Ctx, length(b)::Int64, o::Ref{GmresOpts}, h::Ref{Ptr{Cvoid}})::Int32)
    c = GmresCache(h[], length(b))
    finalizer(x -> (@ccall libb200.b200_gmres_destroy(x.handle::Ptr{Cvoid})::Int32), c)
    return c
end

# host callback used when the operator is an arbitrary SciMLOperator: mul!(y, A, x) on device vectors.  `user` points at a
# `Base.RefValue{Any}` that the caller keeps alive (GC.@preserve) for the duration of the solve.
function _matvec_trampoline(user::Ptr{Cvoid}, x::Ptr{Float64}, y::Ptr{Float64})::Int32
    try
        box = unsafe_pointer_to_objref(user)::Base.RefValue{Any}
        A, ctx, n = box[]::Tuple{Any, Context, Int}
        mul!(unsafe_wrap_device(ctx, y, n), A, unsafe_wrap_device(ctx, x, n))
        return Int32(0)
    catch
        return Int32(1)       # no exception may cross the ABI
    end
end

function SciMLBase.solve!(cache::LinearSolve.LinearCache, alg::B200GMRES; kwargs...)
    gm = cache.cacheval::GmresCache
    b, x, A = cache.b::B200Vector, cache.u::B200Vector, cache.A
    ctx = b.ctx
    check(ctx.handle, @ccall libb200.b200_gmres_set_tolerances(gm.handle::Ptr{Cvoid}, Float64(cache.abstol)::Float64, Float64(cache.reltol)::Float64)::Int32)
    op = Ref{Ptr{Cvoid}}(C_NULL)
    prob = device_problem(A)                       # non-nothing when f.jvp is one of our callables
    ulin = linearisation_point(A)
    ulin === nothing && cache.p isa NonlinearSolveBase.LinearSolveParameters && (ulin = cache.p.u)   # linear_solve.jl:1-4
    box = Ref{Any}((A, ctx, length(b)))
    if prob !== nothing && ulin isa B200Vector
        check(ctx.handle, @ccall libb200.b200_linop_from_problem(prob.handle::Ptr{Cvoid}, vec(ulin).ptr::Ptr{Float64}, 0::Int32, op::Ref{Ptr{Cvoid}})::Int32)
    else
        cb = @cfunction(_matvec_trampoline, Int32, (Ptr{Cvoid}, Ptr{Float64}, Ptr{Float64}))
        check(ctx.handle, @ccall libb200.b200_linop_from_callback(ctx.handle::Ctx, length(b)::Int64, cb::Ptr{Cvoid}, pointer_from_objref(box)::Ptr{Cvoid}, op::Ref{Ptr{Cvoid}})::Int32)
    end
    # LinearSolve `precs`: cache.Pl / cache.Pr.  The marker types map to the library's built-in device preconditioners.
    pl = cache.Pl isa B200Preconditioner && prob !== nothing ? precond_op(cache.Pl, prob, vec(ulin)) : C_NULL
    pr = cache.Pr isa B200Preconditioner && prob !== nothing ? precond_op(cache.Pr, prob, vec(ulin)) : C_NULL
    st = Ref{GmresStats}()
    status = Int32(0)
    GC.@preserve box st begin
        check(ctx.handle, @ccall libb200.b200_gmres_set_precond(gm.handle::Ptr{Cvoid}, pl::Ptr{Cvoid}, pr::Ptr{Cvoid})::Int32)
        status = @ccall libb200.b200_gmres_solve(gm.handle::Ptr{Cvoid}, op[]::Ptr{Cvoid}, b.ptr::Ptr{Float64}, x.ptr::Ptr{Float64}, st::Ref{GmresStats})::Int32
        @ccall libb200.b200_gmres_set_precond(gm.handle::Ptr{Cvoid}, C_NULL::Ptr{Cvoid}, C_NULL::Ptr{Cvoid})::Int32
        @ccall libb200.b200_linop_destroy(op[]::Ptr{Cvoid})::Int32
        pl == C_NULL || @ccall libb200.b200_linop_destroy(pl::Ptr{Cvoid})::Int32
        pr == C_NULL || @ccall libb200.b200_linop_destroy(pr::Ptr{Cvoid})::Int32
    end
    check(ctx.handle, status)
    s = st[]
    rc = s.status == 1 || s.status == 3 ? ReturnCode.Success : s.status == 2 ? ReturnCode.MaxIters : ReturnCode.Failure
    return SciMLBase.build_linear_solution(alg, x, s.rnorm, cache; retcode = rc, iters = Int(s.iters))
end

"""`precs = (A, p) -> (B200BlockJacobi(), I)` / `(I, B200Multigrid())`: the library's built-in preconditioners of the
Brusselator Jacobian (large_systems.md:244-316 hands IncompleteLU.ilu / AlgebraicMultigrid hierarchies to GMRES the same way)."""
abstract type B200Preconditioner end
struct B200BlockJacobi <: B200Preconditioner end
struct B200Multigrid <: B200Preconditioner end
"""`B200ILU0()`: incomplete LU with zero fill of the assembled sparse Jacobian.  It factors the concrete matrix, so it is offered
on the whole-solve path only: `B200NewtonKrylov(; linsolve = :sparse_gmres, precs = :ilu0_left | :ilu0_right)`."""
struct B200ILU0 <: B200Preconditioner end
"""`B200AMG()`: one Ruge-Stueben algebraic-multigrid V-cycle of the assembled sparse Jacobian (Jacobi smoothing).  It coarsens
the concrete matrix, so it is offered on the whole-solve path only: `B200NewtonKrylov(; linsolve = :sparse_gmres,
precs = :amg_left | :amg_right)`; `AMGHierarchy` is the stand-alone handle."""
struct B200AMG <: B200Preconditioner end
"""`B200SAAMG()`: the same with smoothed aggregation, its whole rebuild on the device: `B200NewtonKrylov(; linsolve = :sparse_gmres,
precs = :sa_amg_left | :sa_amg_right)`; `AMGHierarchy(ctx, A; method = :smoothed_aggregation)` is the stand-alone handle."""
struct B200SAAMG <: B200Preconditioner end
precond_kind(::B200BlockJacobi) = Int32(1)      # B200_PRECOND_BLOCK_JACOBI_LEFT (LEFT / RIGHT of a family name the same operator)
precond_kind(::B200Multigrid) = Int32(3)        # B200_PRECOND_MULTIGRID_LEFT
precond_op(::B200ILU0, ::Problem, ::B200Vector) = throw(ArgumentError(
    "B200ILU0 needs the concrete sparse Jacobian: use B200NewtonKrylov(; linsolve = :sparse_gmres, precs = :ilu0_left) (or :ilu0_right)"))
precond_op(::B200AMG, ::Problem, ::B200Vector) = throw(ArgumentError(
    "B200AMG needs the concrete sparse Jacobian: use B200NewtonKrylov(; linsolve = :sparse_gmres, precs = :amg_left) (or :amg_right)"))
precond_op(::B200SAAMG, ::Problem, ::B200Vector) = throw(ArgumentError(
    "B200SAAMG needs the concrete sparse Jacobian: use B200NewtonKrylov(; linsolve = :sparse_gmres, precs = :sa_amg_left) (or :sa_amg_right)"))
function precond_op(P::B200Preconditioner, prob::Problem, u::B200Vector)
    op = Ref{Ptr{Cvoid}}(C_NULL)
    check(prob.ctx.handle, @ccall libb200.b200_linop_precond(prob.handle::Ptr{Cvoid}, u.ptr::Ptr{Float64}, precond_kind(P)::Int32, op::Ref{Ptr{Cvoid}})::Int32)
    return op[]
end

# ------------------------------------------------------------------ algebraic multigrid of an assembled CSC matrix (b200_amg_*)
struct AmgOpts
    theta::Float64
    omega::Float64
    presweeps::Int32
    postsweeps::Int32
    max_levels::Int32
    max_coarse::Int32
end
function default_amg_opts()
    o = Ref{AmgOpts}()
    @ccall libb200.b200_amg_opts_default(o::Ref{AmgOpts})::Cvoid
    return o[]
end
struct SaOpts
    theta::Float64
    omega::Float64
    presweeps::Int32
    postsweeps::Int32
    max_levels::Int32
    max_coarse::Int32
    smooth_omega::Float64
end
function default_sa_opts()
    o = Ref{SaOpts}()
    @ccall libb200.b200_sa_opts_default(o::Ref{SaOpts})::Cvoid
    return o[]
end

"""`AMGHierarchy(ctx, A::SparseMatrixCSC; method = :ruge_stuben | :smoothed_aggregation, opts)`: the device algebraic-multigrid
hierarchy of A's pattern (`opts` an `AmgOpts`, default `default_amg_opts()`, or with smoothed aggregation an `SaOpts`, default
`default_sa_opts()`).  `setup!(h, nzval; rebuild = true)` returns 0 or the 1-based level of a zero diagonal / pivot; `ldiv!(x, h, b)`
applies one V-cycle; `amg_levels(h)` the unknowns and nonzeros per level."""
mutable struct AMGHierarchy
    ctx::Context
    handle::Ptr{Cvoid}
    n::Int
    function AMGHierarchy(ctx::Context, A::SparseMatrixCSC; method::Symbol = :ruge_stuben,
                          opts::Union{AmgOpts, SaOpts} = method === :smoothed_aggregation ? default_sa_opts() : default_amg_opts())
        n = size(A, 1)
        h = Ref{Ptr{Cvoid}}(C_NULL)
        colptr, rowval = Vector{Int64}(A.colptr), Vector{Int64}(A.rowval)
        if method === :smoothed_aggregation
            opts isa SaOpts || throw(ArgumentError("method = :smoothed_aggregation takes SaOpts"))
            check(ctx.handle, @ccall libb200.b200_amg_create_sa(ctx.handle::Ctx, n::Int64, colptr::Ptr{Int64}, rowval::Ptr{Int64}, 1::Int32, Ref(opts)::Ref{SaOpts},
                                                                h::Ref{Ptr{Cvoid}})::Int32)
        elseif method === :ruge_stuben
            opts isa AmgOpts || throw(ArgumentError("method = :ruge_stuben takes AmgOpts"))
            check(ctx.handle, @ccall libb200.b200_amg_create(ctx.handle::Ctx, n::Int64, colptr::Ptr{Int64}, rowval::Ptr{Int64}, 1::Int32, Ref(opts)::Ref{AmgOpts},
                                                             h::Ref{Ptr{Cvoid}})::Int32)
        else
            throw(ArgumentError("method must be :ruge_stuben or :smoothed_aggregation"))
        end
        H = new(ctx, h[], n)
        finalizer(x -> (@ccall libb200.b200_amg_destroy(x.handle::Ptr{Cvoid})::Int32), H)
        return H
    end
end
function setup!(H::AMGHierarchy, nzval::B200Vector; rebuild::Bool = true)
    info = Ref{Int32}(0)
    check(H.ctx.handle, @ccall libb200.b200_amg_setup(H.handle::Ptr{Cvoid}, nzval.ptr::Ptr{Float64}, Int32(rebuild)::Int32, info::Ref{Int32})::Int32)
    return Int(info[])
end
LinearAlgebra.ldiv!(x::B200Vector, H::AMGHierarchy, b::B200Vector) =
    (check(H.ctx.handle, @ccall libb200.b200_amg_solve(H.handle::Ptr{Cvoid}, b.ptr::Ptr{Float64}, x.ptr::Ptr{Float64})::Int32); x)
function amg_levels(H::AMGHierarchy)
    nl = Ref{Int32}(0)
    ns, nz = zeros(Int64, 64), zeros(Int64, 64)
    check(H.ctx.handle, @ccall libb200.b200_amg_levels(H.handle::Ptr{Cvoid}, nl::Ref{Int32}, ns::Ptr{Int64}, nz::Ptr{Int64}, 64::Int32)::Int32)
    return ns[1:nl[]], nz[1:nl[]]
end
"""`amg_split(A::SparseMatrixCSC; theta = 0.25)`: the level-0 C/F splitting on the host (true at C points), no device."""
function amg_split(A::SparseMatrixCSC; theta::Real = 0.25)
    n = size(A, 1)
    cf, nc = zeros(Int32, n), Ref{Int64}(0)
    st = @ccall libb200.b200_amg_split(n::Int64, Vector{Int64}(A.colptr)::Ptr{Int64}, Vector{Int64}(A.rowval)::Ptr{Int64}, Vector{Float64}(A.nzval)::Ptr{Float64},
                                       1::Int32, Float64(theta)::Float64, cf::Ptr{Int32}, nc::Ref{Int64})::Int32
    st == 0 || throw(B200Error(st, "b200_amg_split failed"))
    return cf .== 1
end

# ------------------------------------------------------------------ whole-solve fast path
"""
    B200NewtonKrylov(; problem, linsolve = :gmres | :dense_lu | :sparse_gmres | :sparse_lu,
                       globalization = :none | :trust_region | :linesearch,
                       descent = :newton | :pseudo_transient | :levenberg_marquardt | :broyden,
                       forcing = false, precs = :none | :block_jacobi_left | ... , orth = :mgs)

New `AbstractNonlinearSolveAlgorithm` whose `__solve` runs the entire Newton iteration inside the library
(`b200_newton_*`) and returns `SciMLBase.build_solution(prob, alg, u, resid; retcode, stats = NLStats(nf, njacs, nfactors,
nsolve, nsteps), original)`, as the wrapper algorithms in the reference do (ext/NonlinearSolvePETScExt.jl:162-166).
"""
Base.@kwdef struct B200NewtonKrylov <: NonlinearSolveBase.AbstractNonlinearSolveAlgorithm
    problem::Problem
    linsolve::Symbol = :gmres
    globalization::Symbol = :none
    radius_update_scheme::Symbol = :simple  # :simple | :nlsolve | :nocedal_wright | :hei | :yuan | :fan | :bastin
    descent::Symbol = :newton
    alpha_initial::Float64 = 1.0e-3      # PseudoTransient(alpha_initial)
    forcing::Bool = false                # EisenstatWalkerForcing2()
    precs::Symbol = :none
    orth::Symbol = :mgs
    termination::Symbol = :abs_norm_safe_best
    termination_norm::Symbol = :inf      # internalnorm of the termination mode: :inf (maximum(abs, .)) or :l2
    init_jacobian::Symbol = :identity    # descent = :broyden — Broyden(; init_jacobian = Val(:identity) | Val(:true_jacobian)); :low_rank = LimitedMemoryBroyden
    threshold::Int = 10                  #                      LimitedMemoryBroyden(; threshold = Val(10))
    update_rule::Symbol = :good_broyden  #                      Broyden(; update_rule = Val(:good_broyden) | Val(:bad_broyden))
    max_resets::Int = 100
end

const _LINSOLVE = (gmres = 0, dense_lu = 1, sparse_gmres = 2, sparse_lu = 3)
const _GLOBALIZATION = (none = 0, trust_region = 1, linesearch = 2)
const _DESCENT = (newton = 0, pseudo_transient = 1, levenberg_marquardt = 2, broyden = 3)
const _QN_INIT = (identity = 0, true_jacobian = 1, low_rank = 2)
const _QN_UPDATE = (good_broyden = 0, bad_broyden = 1, klement = 2)
const _TR_SCHEMES = (simple = 0, nlsolve = 1, nocedal_wright = 2, hei = 3, yuan = 4, fan = 5, bastin = 6)
const _PRECS = (none = 0, block_jacobi_left = 1, block_jacobi_right = 2, multigrid_left = 3, multigrid_right = 4, ilu0_left = 5, ilu0_right = 6, amg_left = 7,
    amg_right = 8, sa_amg_left = 9, sa_amg_right = 10)
const _TERMINATION = (abs_norm_safe_best = 0, abs_norm = 1, abs_norm_safe = 2, norm = 3, rel = 4, rel_norm = 5, abs = 6,
    rel_norm_safe = 7, rel_norm_safe_best = 8)

function newton_opts(alg::B200NewtonKrylov; abstol = nothing, reltol = nothing, maxiters = 1000, maxtime = nothing, store_trace = false)
    o = default_newton_opts()
    g = with(o.gmres; orth = orth_code(alg.orth), atol = 0.0, rtol = 0.0)      # inherit the nonlinear tolerances (solve.jl:203)
    return with(o; abstol = something(abstol, 0.0), reltol = something(reltol, 0.0), maxiters = maxiters,
        maxtime = something(maxtime, 0.0), store_trace = store_trace ? 1 : 0, gmres = g,
        linsolve = getfield(_LINSOLVE, alg.linsolve), globalization = getfield(_GLOBALIZATION, alg.globalization),
        forcing = alg.forcing ? 1 : 0, precond = getfield(_PRECS, alg.precs), descent = getfield(_DESCENT, alg.descent),
        tr_scheme = getfield(_TR_SCHEMES, alg.radius_update_scheme), pt_alpha_initial = alg.alpha_initial,
        termination = getfield(_TERMINATION, alg.termination), term_norm = alg.termination_norm === :l2 ? 1 : 0,
        qn_init_jacobian = getfield(_QN_INIT, alg.init_jacobian), qn_update_rule = getfield(_QN_UPDATE, alg.update_rule),
        qn_max_resets = alg.max_resets, qn_threshold = alg.threshold)
end

function SciMLBase.__solve(prob::SciMLBase.NonlinearProblem, alg::B200NewtonKrylov, args...;
        abstol = nothing, reltol = nothing, maxiters = 1000, maxtime = nothing, kwargs...)
    dp, ctx = alg.problem, alg.problem.ctx
    o = Ref(newton_opts(alg; abstol, reltol, maxiters, maxtime))
    nw = Ref{Ptr{Cvoid}}(C_NULL)
    check(ctx.handle, @ccall libb200.b200_newton_create(dp.handle::Ptr{Cvoid}, o::Ref{NewtonOpts}, nw::Ref{Ptr{Cvoid}})::Int32)
    try
        res = Ref{NewtonResult}()
        u0 = prob.u0
        if u0 isa B200Vector
            check(ctx.handle, @ccall libb200.b200_newton_reinit(nw[]::Ptr{Cvoid}, u0.ptr::Ptr{Float64})::Int32)
            check(ctx.handle, @ccall libb200.b200_newton_solve(nw[]::Ptr{Cvoid}, res::Ref{NewtonResult})::Int32)
            pu = Ref{Ptr{Float64}}(C_NULL); pf = Ref{Ptr{Float64}}(C_NULL)
            check(ctx.handle, @ccall libb200.b200_newton_u(nw[]::Ptr{Cvoid}, pu::Ref{Ptr{Float64}})::Int32)
            check(ctx.handle, @ccall libb200.b200_newton_fu(nw[]::Ptr{Cvoid}, pf::Ref{Ptr{Float64}})::Int32)
            u = copy(unsafe_wrap_device(ctx, pu[], dp.n)); fu = copy(unsafe_wrap_device(ctx, pf[], dp.n))   # copies outlive the cache
        else    # host arrays: the end-to-end call (H2D, solve, D2H)
            u0h = vec(collect(Float64, u0)); u = similar(u0h); fu = similar(u0h)
            GC.@preserve u0h u fu check(ctx.handle, @ccall libb200.b200_newton_solve_host(nw[]::Ptr{Cvoid}, pointer(u0h)::Ptr{Float64},
                pointer(u)::Ptr{Float64}, pointer(fu)::Ptr{Float64}, res::Ref{NewtonResult})::Int32)
            u = reshape(u, size(u0)); fu = reshape(fu, size(u0))
        end
        r = res[]
        stats = NLStats(Int(r.nf), Int(r.njacs), Int(r.nfactors), Int(r.nsolve), Int(r.nsteps))
        return SciMLBase.build_solution(prob, alg, u, fu; retcode = retcode(r.retcode), stats, original = r)
    finally
        @ccall libb200.b200_newton_destroy(nw[]::Ptr{Cvoid})::Int32
    end
end

# ------------------------------------------------------------------ b6: ensemble algorithm
"""
    EnsembleB200(; rank = 0, world_size = 1, unique_id = nothing, gather = true)

`solve(ensembleprob, alg, EnsembleB200(); trajectories)` evaluates `prob_func(prob, i, repeat)` for the trajectories of
this rank's contiguous block, packs `u0` / `(A, B)` into batches and calls `b200_ens_solve` (one CTA per trajectory, no
collective on the data path).  `alg`'s `NewtonOpts.globalization` is forwarded: undamped Newton, the BackTracking line search
and the trust region (Dogleg) are batched, the latter two without a preconditioner (`b200_ens_create` refuses a globalised
ensemble with one).  With `world_size > 1` (one process per GPU) the solutions of all ranks are collected in
trajectory order by `b200_ens_allgather` and the status counters by `b200_ens_allreduce_stats` — NCCL over NVLink inside
the library; `unique_id` is the 128-byte id from `nccl_unique_id()` on rank 0, shipped by the launcher (MPI.bcast, a file).
"""
Base.@kwdef struct EnsembleB200 <: SciMLBase.EnsembleAlgorithm
    rank::Int = 0
    world_size::Int = 1
    unique_id::Union{Nothing, Vector{UInt8}} = nothing
    gather::Bool = true
end
function nccl_unique_id()
    id = zeros(UInt8, 128)
    GC.@preserve id check(C_NULL, @ccall libb200.b200_nccl_unique_id(pointer(id)::Ptr{Cvoid})::Int32)
    return id
end

function shard_range(K::Integer, rank::Integer, world::Integer)
    base, rem = divrem(K, world)
    lo = rank * base + min(rank, rem)
    return (lo + 1):(lo + base + (rank < rem ? 1 : 0))      # 1-based trajectory indices of this rank
end
_prob_func(ens, i) = applicable(ens.prob_func, ens.prob, i, 1) ? ens.prob_func(ens.prob, i, 1) : ens.prob_func(ens.prob, (; sim_id = i, repeat = 1))  # both forms of core_tests__item6.jl:3-4

function SciMLBase.__solve(ens::SciMLBase.AbstractEnsembleProblem, alg::B200NewtonKrylov, ealg::EnsembleB200; trajectories, abstol = nothing, reltol = nothing,
        maxiters = 1000, kwargs...)
    ctx = alg.problem.ctx
    t0 = time()
    idx = shard_range(trajectories, ealg.rank, ealg.world_size)
    probs = [_prob_func(ens, i) for i in idx]
    N = round(Int, sqrt(length(first(probs).u0) ÷ 2)); n = 2N^2; K = length(idx)
    u0 = reduce(hcat, (vec(collect(Float64, p.u0)) for p in probs)); A = Float64[p.p[1] for p in probs]; B = Float64[p.p[2] for p in probs]
    d_u0, d_A, d_B, d_u = B200Vector(ctx, u0), B200Vector(ctx, A), B200Vector(ctx, B), B200Vector(ctx, n * K)
    d_res = B200Vector(ctx, K)
    d_rc, d_ns, d_nj = DeviceBuffer{Int32}(ctx, K), DeviceBuffer{Int32}(ctx, K), DeviceBuffer{Int32}(ctx, K)
    o = Ref(newton_opts(alg; abstol, reltol, maxiters))
    h = Ref{Ptr{Cvoid}}(C_NULL)
    check(ctx.handle, @ccall libb200.b200_ens_create(ctx.handle::Ctx, N::Int32, K::Int32, Float64(first(probs).p[3])::Float64, o::Ref{NewtonOpts}, h::Ref{Ptr{Cvoid}})::Int32)
    local_res = Ref{EnsResult}()
    try
        check(ctx.handle, @ccall libb200.b200_ens_solve(h[]::Ptr{Cvoid}, d_u0.ptr::Ptr{Float64}, d_A.ptr::Ptr{Float64}, d_B.ptr::Ptr{Float64}, d_u.ptr::Ptr{Float64},
            d_res.ptr::Ptr{Float64}, d_rc.ptr::Ptr{Int32}, d_ns.ptr::Ptr{Int32}, d_nj.ptr::Ptr{Int32}, local_res::Ref{EnsResult})::Int32)
    finally
        @ccall libb200.b200_ens_destroy(h[]::Ptr{Cvoid})::Int32
    end
    U = reshape(Array(d_u), n, K)
    rcs, nss, resid = Array(d_rc), Array(d_ns), Array(d_res)
    # per-trajectory residual vectors f(u_k; A_k, B_k) for `sol.resid` (one cheap stencil launch each)
    F = similar(U)
    tmp_u, tmp_f = B200Vector(ctx, n), B200Vector(ctx, n)
    for k in 1:K
        check(ctx.handle, @ccall libb200.b200_problem_set_AB(alg.problem.handle::Ptr{Cvoid}, A[k]::Float64, B[k]::Float64)::Int32)
        copyto!(tmp_u, U[:, k]); residual!(tmp_f, tmp_u, alg.problem)
        F[:, k] = Array(tmp_f)
    end
    sols = [SciMLBase.build_solution(probs[k], alg, reshape(U[:, k], size(probs[k].u0)), reshape(F[:, k], size(probs[k].u0));
                retcode = retcode(rcs[k]), stats = NLStats(Int(nss[k]), 0, 0, Int(nss[k]), Int(nss[k])), original = resid[k]) for k in 1:K]
    converged = all(SciMLBase.successful_retcode(s.retcode) for s in sols)
    if ealg.world_size > 1 && ealg.gather
        ealg.unique_id === nothing && throw(ArgumentError("EnsembleB200(world_size > 1) needs the unique_id created by nccl_unique_id() on rank 0"))
        trajectories % ealg.world_size == 0 || throw(ArgumentError("the gather needs equal blocks: trajectories must be a multiple of world_size"))
        id = ealg.unique_id
        comm = Ref{Ptr{Cvoid}}(C_NULL)
        GC.@preserve id check(ctx.handle, @ccall libb200.b200_nccl_init(ctx.handle::Ctx, ealg.world_size::Int32, ealg.rank::Int32, pointer(id)::Ptr{Cvoid}, comm::Ref{Ptr{Cvoid}})::Int32)
        d_all = B200Vector(ctx, n * trajectories)
        global_res = Ref{EnsResult}()
        try
            check(ctx.handle, @ccall libb200.b200_ens_allgather(comm[]::Ptr{Cvoid}, d_u.ptr::Ptr{Float64}, (n * K)::Int64, d_all.ptr::Ptr{Float64})::Int32)
            check(ctx.handle, @ccall libb200.b200_ens_allreduce_stats(comm[]::Ptr{Cvoid}, local_res::Ref{EnsResult}, global_res::Ref{EnsResult})::Int32)
        finally
            @ccall libb200.b200_nccl_destroy(comm[]::Ptr{Cvoid})::Int32
        end
        Uall = reshape(Array(d_all), n, trajectories)
        # trajectories of the other ranks: solution and the globally reduced verdict (their per-trajectory stats stay with their rank)
        sols = [k in idx ? sols[k - first(idx) + 1] :
                SciMLBase.build_solution(first(probs), alg, reshape(Uall[:, k], size(first(probs).u0)), nothing; retcode = ReturnCode.Default) for k in 1:trajectories]
        converged = global_res[].nsuccess == global_res[].nprob
    end
    return SciMLBase.EnsembleSolution(sols, time() - t0, converged)
end

export Context, B200Vector, brusselator, brusselator_function, initial_condition, B200GMRES, B200BlockJacobi, B200Multigrid, B200ILU0, B200AMG, B200SAAMG, AMGHierarchy, setup!, amg_levels, amg_split,
    B200NewtonKrylov, EnsembleB200, nccl_unique_id, device_count

end # module
