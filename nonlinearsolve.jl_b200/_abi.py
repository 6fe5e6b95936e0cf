"""ctypes binding of include/b200newton.h (the C ABI of libb200newton.so).

This is the same call sequence the Julia glue (julia/B200Newton) issues through `@ccall`; see INTEGRATION.md.
There is no CPU fallback: if the shared library is missing, or no CUDA device is present when a context is
created, an exception is raised.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200newton.so")

# ---- enums (include/b200newton.h)
OK, ERR_CUDA, ERR_INVALID, ERR_NOMEM, ERR_UNSUPPORTED, ERR_CALLBACK, ERR_NO_DEVICE = 0, -1, -2, -3, -4, -5, -6
RC_DEFAULT, RC_SUCCESS, RC_MAXITERS, RC_MAXTIME, RC_STALLED, RC_STALLED_SUCCESS, RC_UNSTABLE = 0, 1, 2, 3, 4, 5, 6
RC_INTERNAL_LINSOLVE_FAILED, RC_INTERNAL_LINESEARCH_FAILED, RC_SHRINK_THRESHOLD_EXCEEDED, RC_INITIAL_FAILURE, RC_FAILURE = 7, 8, 9, 10, 11
RC_CONVERGENCE_FAILURE = 12
RETCODE_NAMES = {0: "Default", 1: "Success", 2: "MaxIters", 3: "MaxTime", 4: "Stalled", 5: "StalledSuccess", 6: "Unstable",
                 7: "InternalLinearSolveFailed", 8: "InternalLineSearchFailed", 9: "ShrinkThresholdExceeded",
                 10: "InitialFailure", 11: "Failure", 12: "ConvergenceFailure"}
LS_SOLVED, LS_MAXITERS, LS_BREAKDOWN, LS_NONFINITE, LS_OUT_OF_MEMORY = 1, 2, 3, 4, 5
PROB_BRUSS2D, PROB_BRUSS3D, PROB_QUADRATIC, PROB_TRIDIAG_QUAD, PROB_CALLBACK = 1, 2, 3, 4, 5
ORTH_MGS, ORTH_CGS, ORTH_CGS2 = 0, 1, 2
ENGINE_AUTO, ENGINE_MULTIKERNEL, ENGINE_RESIDENT = 0, 1, 2
LINSOLVE_GMRES, LINSOLVE_DENSE_LU, LINSOLVE_SPARSE_GMRES, LINSOLVE_SPARSE_LU = 0, 1, 2, 3
JVP_EXACT, JVP_FINITE_DIFF = 0, 1
GLOB_NONE, GLOB_TRUST_REGION, GLOB_LINESEARCH = 0, 1, 2
PRECOND_NONE, PRECOND_BLOCK_JACOBI_LEFT, PRECOND_BLOCK_JACOBI_RIGHT, PRECOND_MULTIGRID_LEFT, PRECOND_MULTIGRID_RIGHT = 0, 1, 2, 3, 4
PRECOND_ILU0_LEFT, PRECOND_ILU0_RIGHT = 5, 6
PRECOND_AMG_LEFT, PRECOND_AMG_RIGHT = 7, 8
PRECOND_SA_AMG_LEFT, PRECOND_SA_AMG_RIGHT = 9, 10
AMG_EXPORT_A, AMG_EXPORT_P, AMG_EXPORT_T = 0, 1, 2
DESCENT_NEWTON, DESCENT_PSEUDO_TRANSIENT, DESCENT_LEVENBERG_MARQUARDT, DESCENT_BROYDEN = 0, 1, 2, 3
QN_INIT_IDENTITY, QN_INIT_TRUE_JACOBIAN, QN_INIT_LOW_RANK = 0, 1, 2
QN_UPDATE_GOOD_BROYDEN, QN_UPDATE_BAD_BROYDEN, QN_UPDATE_KLEMENT = 0, 1, 2
TR_SIMPLE, TR_NLSOLVE, TR_NOCEDAL_WRIGHT, TR_HEI, TR_YUAN, TR_FAN, TR_BASTIN = range(7)
FORCING_NONE, FORCING_EW2 = 0, 1
TERM_ABS_NORM_SAFE_BEST, TERM_ABS_NORM, TERM_ABS_NORM_SAFE, TERM_NORM, TERM_REL, TERM_REL_NORM, TERM_ABS, TERM_REL_NORM_SAFE, TERM_REL_NORM_SAFE_BEST = range(9)
NORM_INF, NORM_L2 = 0, 1
U0_REFERENCE, U0_PERTURBED_Z = 0, 1
ORDER_NATURAL, ORDER_LARGEST_FIRST = 0, 1
KID_NAMES = ["jvp", "multidot", "update", "mgs", "normalize", "residual", "givens", "resident", "lu_panel", "lu_gemm", "lu_other", "sparse"]


class GmresOpts(C.Structure):
    _fields_ = [("memory", C.c_int32), ("restart", C.c_int32), ("itmax", C.c_int32), ("orth", C.c_int32),
                ("warm_start", C.c_int32), ("engine", C.c_int32), ("check_every", C.c_int32), ("block", C.c_int32),
                ("atol", C.c_double), ("rtol", C.c_double)]


class GmresStats(C.Structure):
    _fields_ = [("status", C.c_int32), ("iters", C.c_int32), ("nmatvec", C.c_int32), ("restarts", C.c_int32),
                ("rnorm0", C.c_double), ("rnorm", C.c_double), ("tol", C.c_double), ("bytes", C.c_double)]


class NewtonOpts(C.Structure):
    _fields_ = [("abstol", C.c_double), ("reltol", C.c_double), ("maxiters", C.c_int32), ("linsolve", C.c_int32),
                ("jvp_mode", C.c_int32), ("globalization", C.c_int32), ("forcing", C.c_int32), ("termination", C.c_int32),
                ("store_trace", C.c_int32), ("fused_step", C.c_int32), ("gmres", GmresOpts),
                ("ew_eta0", C.c_double), ("ew_eta_max", C.c_double), ("ew_gamma", C.c_double), ("ew_alpha", C.c_double),
                ("ew_safeguard_threshold", C.c_double), ("ew_safeguard", C.c_int32), ("max_shrink_times", C.c_int32),
                ("tr_step_threshold", C.c_double), ("tr_shrink_threshold", C.c_double), ("tr_expand_threshold", C.c_double),
                ("tr_shrink_factor", C.c_double), ("tr_expand_factor", C.c_double), ("tr_max_trust_radius", C.c_double),
                ("tr_initial_trust_radius", C.c_double), ("ls_c1", C.c_double), ("ls_rho_hi", C.c_double), ("ls_rho_lo", C.c_double),
                ("ls_maxiters", C.c_int32), ("precond", C.c_int32), ("descent", C.c_int32), ("tr_scheme", C.c_int32),
                ("pt_alpha_initial", C.c_double), ("maxtime", C.c_double), ("term_norm", C.c_int32), ("term_max_stalled_steps", C.c_int32),
                ("lm_damping_initial", C.c_double), ("lm_damping_increase", C.c_double), ("lm_damping_decrease", C.c_double), ("lm_finite_diff_step", C.c_double),
                ("lm_alpha_geodesic", C.c_double), ("lm_b_uphill", C.c_double), ("lm_min_damping_D", C.c_double), ("lm_disable_geodesic", C.c_int32),
                ("reserved0", C.c_int32),
                ("qn_init_jacobian", C.c_int32), ("qn_update_rule", C.c_int32), ("qn_max_resets", C.c_int32), ("qn_threshold", C.c_int32),
                ("qn_reset_tolerance", C.c_double), ("qn_alpha", C.c_double)]


class NewtonResult(C.Structure):
    _fields_ = [("retcode", C.c_int32), ("nsteps", C.c_int32), ("nf", C.c_int32), ("njacs", C.c_int32),
                ("nfactors", C.c_int32), ("nsolve", C.c_int32), ("njvp", C.c_int32), ("ntrace", C.c_int32),
                ("resid_inf", C.c_double), ("bytes", C.c_double)]


class TraceRec(C.Structure):
    _fields_ = [("iter", C.c_int32), ("lin_iters", C.c_int32), ("lin_status", C.c_int32), ("accepted", C.c_int32),
                ("fnorm_inf", C.c_double), ("step_norm2", C.c_double), ("lin_rnorm", C.c_double), ("trust_radius", C.c_double)]


class EnsResult(C.Structure):
    _fields_ = [("nprob", C.c_int32), ("nsuccess", C.c_int32), ("max_nsteps", C.c_int32), ("reserved", C.c_int32),
                ("total_nsteps", C.c_int64), ("total_njvp", C.c_int64), ("worst_resid_inf", C.c_double)]


class AmgOpts(C.Structure):
    _fields_ = [("theta", C.c_double), ("omega", C.c_double), ("presweeps", C.c_int32), ("postsweeps", C.c_int32),
                ("max_levels", C.c_int32), ("max_coarse", C.c_int32)]


class SaOpts(C.Structure):
    _fields_ = [("theta", C.c_double), ("omega", C.c_double), ("presweeps", C.c_int32), ("postsweeps", C.c_int32),
                ("max_levels", C.c_int32), ("max_coarse", C.c_int32), ("smooth_omega", C.c_double)]


RESIDUAL_CB = C.CFUNCTYPE(C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p)
JVP_CB = C.CFUNCTYPE(C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p)
MATVEC_CB = C.CFUNCTYPE(C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p)
JAC_CB = C.CFUNCTYPE(C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p)

P = C.c_void_p
PP = C.POINTER(C.c_void_p)
I32, I64, F64, SZ = C.c_int32, C.c_int64, C.c_double, C.c_size_t
PI32, PI64, PF64 = C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_double)

# every symbol include/b200newton.h declares: name -> (restype, argtypes)
SIGNATURES = {
    "b200_version": (I32, []),
    "b200_device_count": (I32, [PI32]),
    "b200_ctx_create": (I32, [I32, P, PP]),
    "b200_ctx_destroy": (I32, [P]),
    "b200_ctx_sync": (I32, [P]),
    "b200_ctx_stream": (P, [P]),
    "b200_last_error": (C.c_char_p, [P]),
    "b200_ctx_kernel_launches": (I32, [P, PI64]),
    "b200_ctx_sm_count": (I32, [P, PI32]),
    "b200_ctx_profile_enable": (I32, [P, I32]),
    "b200_ctx_profile_reset": (I32, [P]),
    "b200_ctx_profile_get": (I32, [P, I32, PF64, PF64, PI64]),
    "b200_malloc": (I32, [P, SZ, PP]),
    "b200_free": (I32, [P, P]),
    "b200_host_alloc": (I32, [P, SZ, PP]),
    "b200_host_free": (I32, [P, P]),
    "b200_memcpy_h2d": (I32, [P, P, P, SZ]),
    "b200_memcpy_d2h": (I32, [P, P, P, SZ]),
    "b200_memcpy_d2d": (I32, [P, P, P, SZ]),
    "b200_memset": (I32, [P, P, I32, SZ]),
    "b200_flush_l2": (I32, [P]),
    "b200_fill": (I32, [P, I64, F64, P]),
    "b200_copy": (I32, [P, I64, P, P]),
    "b200_scal": (I32, [P, I64, F64, P]),
    "b200_axpy": (I32, [P, I64, F64, P, P]),
    "b200_axpby": (I32, [P, I64, F64, P, F64, P]),
    "b200_mul": (I32, [P, I64, P, P, P]),
    "b200_dot": (I32, [P, I64, P, P, PF64]),
    "b200_nrm2": (I32, [P, I64, P, PF64]),
    "b200_norminf": (I32, [P, I64, P, PF64]),
    "b200_diffnrm2": (I32, [P, I64, P, P, PF64]),
    "b200_extrema": (I32, [P, I64, P, PF64, PF64]),
    "b200_equal": (I32, [P, I64, P, P, PI32]),
    "b200_problem_create_bruss2d": (I32, [P, I32, F64, F64, F64, PP]),
    "b200_problem_create_bruss3d": (I32, [P, I32, F64, F64, F64, PP]),
    "b200_problem_create_quadratic": (I32, [P, I64, F64, PP]),
    "b200_problem_create_tridiag_quad": (I32, [P, I64, P, PP]),
    "b200_problem_create_callback": (I32, [P, I64, RESIDUAL_CB, JVP_CB, JVP_CB, P, PP]),
    "b200_problem_set_jac": (I32, [P, JAC_CB, JAC_CB]),
    "b200_problem_set_jac_prototype": (I32, [P, P, P, I32]),
    "b200_problem_destroy": (I32, [P]),
    "b200_problem_n": (I32, [P, PI64]),
    "b200_problem_set_AB": (I32, [P, F64, F64]),
    "b200_problem_u0": (I32, [P, I32, P]),
    "b200_residual": (I32, [P, P, P]),
    "b200_jvp": (I32, [P, P, P, P]),
    "b200_residual_jvp": (I32, [P, P, P, P, P]),
    "b200_jvp_fd": (I32, [P, P, P, P]),
    "b200_vjp": (I32, [P, P, P, P]),
    "b200_linop_from_problem": (I32, [P, P, I32, PP]),
    "b200_linop_from_csc": (I32, [P, I64, P, P, P, I32, PP]),
    "b200_linop_from_dense": (I32, [P, I64, P, I64, PP]),
    "b200_linop_from_callback": (I32, [P, I64, MATVEC_CB, P, PP]),
    "b200_linop_apply": (I32, [P, P, P]),
    "b200_linop_destroy": (I32, [P]),
    "b200_gmres_opts_default": (None, [C.POINTER(GmresOpts)]),
    "b200_gmres_create": (I32, [P, I64, C.POINTER(GmresOpts), PP]),
    "b200_gmres_destroy": (I32, [P]),
    "b200_gmres_set_tolerances": (I32, [P, F64, F64]),
    "b200_gmres_set_precond": (I32, [P, P, P]),
    "b200_linop_set_shift": (I32, [P, F64]),
    "b200_linop_block_jacobi": (I32, [P, P, PP]),
    "b200_linop_precond": (I32, [P, P, I32, PP]),
    "b200_sparse_lu_create": (I32, [P, I64, P, P, I32, PP]),
    "b200_sparse_lu_destroy": (I32, [P]),
    "b200_sparse_lu_bandwidth": (I32, [P, PI64, PI64]),
    "b200_sparse_lu_factor": (I32, [P, P, PI32]),
    "b200_sparse_lu_solve": (I32, [P, P, P]),
    "b200_ilu0_create": (I32, [P, I64, P, P, I32, PP]),
    "b200_ilu0_destroy": (I32, [P]),
    "b200_ilu0_levels": (I32, [P, PI32, PI32]),
    "b200_ilu0_factor": (I32, [P, P, PI32]),
    "b200_ilu0_solve": (I32, [P, P, P]),
    "b200_ilu0_export": (I32, [P, P]),
    "b200_ilu0_linop": (I32, [P, PP]),
    "b200_amg_opts_default": (None, [C.POINTER(AmgOpts)]),
    "b200_amg_create": (I32, [P, I64, P, P, I32, C.POINTER(AmgOpts), PP]),
    "b200_amg_destroy": (I32, [P]),
    "b200_amg_setup": (I32, [P, P, I32, PI32]),
    "b200_amg_solve": (I32, [P, P, P]),
    "b200_amg_levels": (I32, [P, PI32, P, P, I32]),
    "b200_amg_export": (I32, [P, I32, I32, P, P, P]),
    "b200_amg_linop": (I32, [P, PP]),
    "b200_amg_split": (I32, [I64, P, P, P, I32, F64, P, PI64]),
    "b200_sa_opts_default": (None, [C.POINTER(SaOpts)]),
    "b200_amg_create_sa": (I32, [P, I64, P, P, I32, C.POINTER(SaOpts), PP]),
    "b200_gmres_solve": (I32, [P, P, P, P, C.POINTER(GmresStats)]),
    "b200_dense_jac_fill": (I32, [P, P, P, I64]),
    "b200_getrf": (I32, [P, I64, P, I64, P, PI32]),
    "b200_getrs": (I32, [P, I64, I64, P, I64, P, P, I64]),
    "b200_gemv": (I32, [P, I32, I64, I64, P, I64, P, P]),
    "b200_pattern_nnz": (I32, [P, PI64]),
    "b200_pattern": (I32, [P, I32, P, P]),
    "b200_coloring_column": (I32, [I64, P, P, I32, I32, P, PI64]),
    "b200_sparse_jac_create": (I32, [P, P, P, I32, P, I64, PP]),
    "b200_sparse_jac_destroy": (I32, [P]),
    "b200_sparse_jac_fill": (I32, [P, P, P]),
    "b200_sparse_jac_linop": (I32, [P, P, PP]),
    "b200_spmv": (I32, [P, P, P, P]),
    "b200_spmv_t": (I32, [P, P, P, P]),
    "b200_newton_opts_default": (None, [C.POINTER(NewtonOpts)]),
    "b200_newton_create": (I32, [P, C.POINTER(NewtonOpts), PP]),
    "b200_newton_destroy": (I32, [P]),
    "b200_newton_reinit": (I32, [P, P]),
    "b200_newton_step": (I32, [P, PI32]),
    "b200_newton_solve": (I32, [P, C.POINTER(NewtonResult)]),
    "b200_newton_result_get": (I32, [P, C.POINTER(NewtonResult)]),
    "b200_newton_u": (I32, [P, PP]),
    "b200_newton_fu": (I32, [P, PP]),
    "b200_newton_trace": (I32, [P, C.POINTER(TraceRec), I32, PI32]),
    "b200_newton_solve_host": (I32, [P, P, P, P, C.POINTER(NewtonResult)]),
    "b200_ens_create": (I32, [P, I32, I32, F64, C.POINTER(NewtonOpts), PP]),
    "b200_ens_destroy": (I32, [P]),
    "b200_ens_solve": (I32, [P, P, P, P, P, P, P, P, P, C.POINTER(EnsResult)]),
    "b200_ens_precond_apply": (I32, [P, P, P, P, P]),
    "b200_ens_ctas_per_sm": (I32, [P, PI32]),
    "b200_nccl_version": (I32, [PI32]),
    "b200_nccl_unique_id": (I32, [P]),
    "b200_nccl_init": (I32, [P, I32, I32, P, PP]),
    "b200_nccl_init_all": (I32, [PP, I32, PP]),
    "b200_nccl_group_start": (I32, []),
    "b200_nccl_group_end": (I32, []),
    "b200_nccl_destroy": (I32, [P]),
    "b200_ens_allgather": (I32, [P, P, I64, P]),
    "b200_ens_allreduce_stats_begin": (I32, [P, C.POINTER(EnsResult)]),
    "b200_ens_allreduce_stats_finish": (I32, [P, C.POINTER(EnsResult)]),
    "b200_ens_allreduce_stats": (I32, [P, C.POINTER(EnsResult), C.POINTER(EnsResult)]),
}
# test hooks exported by the library but not part of the public header
EXTRA_SIGNATURES = {
    "b200_gmres_keep_hessenberg": (I32, [P, I64]),
    "b200_gmres_get_hessenberg": (I32, [P, P, I64]),
}

_lib = None


class B200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("b200newton error %d: %s" % (code, msg))
        self.code = code


def lib():
    """Load libb200newton.so (fails loudly when it has not been built: there is no fallback path)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError("%s not found: build it with `python nonlinearsolve.jl_b200/build.py` "
                              "(or __graft_entry__.build()); there is no CPU fallback." % LIB_PATH)
        L = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
        for table in (SIGNATURES, EXTRA_SIGNATURES):
            for name, (res, args) in table.items():
                fn = getattr(L, name)
                fn.restype = res
                fn.argtypes = args
        _lib = L
    return _lib


def check(ctx, status):
    if status != OK:
        msg = lib().b200_last_error(ctx).decode() if ctx else ""
        raise B200Error(status, msg)
