/*
 * b200newton.h — C ABI of libb200newton.so, the H100-native (sm_90a) Newton iteration core
 * that sits behind NonlinearSolve.jl's first-order solver plugin points.
 *
 * Every entry point is `extern "C"`, takes plain pointers/sizes and returns an int32 status
 * (0 = B200_OK, negative = infrastructure error, see b200_last_error()).  Numerical outcomes
 * (converged / max-iters / stalled ...) are NOT errors: they come back in result structs as
 * retcodes that map 1:1 onto SciMLBase.ReturnCode.
 *
 * Reference interface each group replaces (paths relative to the NonlinearSolve.jl tree):
 *   problems / residual      user f!(du,u,p)      lib/NonlinearSolveBase/src/utils.jl:180-207
 *                            Brusselator spec     lib/NonlinearSolveFirstOrder/test/sparsity_tests__item1.jl:7-50
 *   jvp / vjp                JacobianOperator     lib/SciMLJacobianOperators/src/SciMLJacobianOperators.jl:167-182, 238-243, 296-431
 *   gmres                    LinearSolveJLCache   lib/NonlinearSolveBase/ext/NonlinearSolveBaseLinearSolveExt.jl:16-32
 *                            (-> LinearSolve.KrylovJL_GMRES -> Krylov.gmres!, external)
 *   dense jac / LU           JacobianCache        lib/NonlinearSolveBase/src/jacobian.jl:237-258
 *                            linear cache         lib/NonlinearSolveBase/src/linear_solve.jl:74-147
 *   sparse pattern/colouring construct_concrete_adtype  lib/NonlinearSolveBase/src/jacobian.jl:286-353
 *                            colouring choice     lib/NonlinearSolveBase/ext/NonlinearSolveBaseSparseMatrixColoringsExt.jl:13-28
 *   newton driver            step!                lib/NonlinearSolveFirstOrder/src/solve.jl:325-465
 *                            termination          lib/NonlinearSolveBase/src/termination_conditions.jl:243-336
 *                            trust region/dogleg  lib/NonlinearSolveFirstOrder/src/trust_region.jl:396-514,
 *                                                 lib/NonlinearSolveBase/src/descent/dogleg.jl:86-151
 *                            forcing              lib/NonlinearSolveFirstOrder/src/eisenstat_walker.jl:42-87
 *   ensemble                 EnsembleProblem use  test/PolyAlgorithms/core_tests__item6.jl:3-20
 *
 * Conventions: all data vectors are Float64 DEVICE pointers unless a parameter name ends in
 * `_host`; small result structs are HOST pointers.  Work is enqueued on the context's stream;
 * calls that return a host scalar/struct synchronise that stream.  A context is not thread-safe.
 * Index arrays are int64 with an explicit `index_base` (Julia: 1).
 */
#ifndef B200NEWTON_H
#define B200NEWTON_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_VERSION 100 /* 0.1.0 */

/* ---------------------------------------------------------------- status codes */
enum {
  B200_OK = 0,
  B200_ERR_CUDA = -1,
  B200_ERR_INVALID = -2,
  B200_ERR_NOMEM = -3,
  B200_ERR_UNSUPPORTED = -4,
  B200_ERR_CALLBACK = -5,
  B200_ERR_NO_DEVICE = -6
};

/* nonlinear-solve return codes; names follow SciMLBase.ReturnCode */
enum {
  B200_RC_DEFAULT = 0,
  B200_RC_SUCCESS = 1,
  B200_RC_MAXITERS = 2,
  B200_RC_MAXTIME = 3,
  B200_RC_STALLED = 4,
  B200_RC_STALLED_SUCCESS = 5,
  B200_RC_UNSTABLE = 6,
  B200_RC_INTERNAL_LINSOLVE_FAILED = 7,
  B200_RC_INTERNAL_LINESEARCH_FAILED = 8,
  B200_RC_SHRINK_THRESHOLD_EXCEEDED = 9,
  B200_RC_INITIAL_FAILURE = 10,
  B200_RC_FAILURE = 11,
  B200_RC_CONVERGENCE_FAILURE = 12 /* quasi-Newton: max_resets reached (NonlinearSolveQuasiNewton/src/solve.jl:343-347) */
};

/* linear (GMRES) solve status; maps to LinearSolve retcodes (Success / MaxIters / Failure) */
enum {
  B200_LS_SOLVED = 1,      /* ||r|| <= atol + rtol*||r0||                    -> ReturnCode.Success  */
  B200_LS_MAXITERS = 2,    /* itmax reached                                    -> ReturnCode.MaxIters */
  B200_LS_BREAKDOWN = 3,   /* happy breakdown, solution exact in the subspace  -> ReturnCode.Success  */
  B200_LS_NONFINITE = 4,   /* NaN/Inf met                                      -> ReturnCode.Failure  */
  B200_LS_OUT_OF_MEMORY = 5 /* Krylov basis could not grow                     -> ReturnCode.Failure  */
};

enum { B200_PROB_BRUSS2D = 1, B200_PROB_BRUSS3D = 2, B200_PROB_QUADRATIC = 3, B200_PROB_TRIDIAG_QUAD = 4, B200_PROB_CALLBACK = 5 };
enum { B200_ORTH_MGS = 0, B200_ORTH_CGS = 1, B200_ORTH_CGS2 = 2 };
enum { B200_ENGINE_AUTO = 0, B200_ENGINE_MULTIKERNEL = 1, B200_ENGINE_RESIDENT = 2 };
/* SPARSE_LU: what NewtonRaphson() does on a sparse jac_prototype (linsolve = nothing -> LinearSolve's sparse direct default,
   KLU/UMFPACK; sparsity_tests__item1.jl:54-93, operator_jacobian.jl:22): coloured sparse Jacobian + a direct factorisation
   (reverse Cuthill-McKee ordering + banded LU with partial pivoting on the device, b200_sparse_lu_*) */
enum { B200_LINSOLVE_GMRES = 0, B200_LINSOLVE_DENSE_LU = 1, B200_LINSOLVE_SPARSE_GMRES = 2, B200_LINSOLVE_SPARSE_LU = 3 };
enum { B200_JVP_EXACT = 0, B200_JVP_FINITE_DIFF = 1 };
enum { B200_GLOBALIZATION_NONE = 0, B200_GLOBALIZATION_TRUST_REGION = 1, B200_GLOBALIZATION_LINESEARCH = 2 };
/* descent: NewtonDescent (descent/newton.jl) or DampedNewtonDescent + SwitchedEvolutionRelaxation = PseudoTransient
   (descent/damped_newton.jl:234-340, NonlinearSolveFirstOrder/src/pseudo_transient.jl:37-170): (J + I/alpha) du = -f */
/* RadiusUpdateSchemes.{Simple, NLsolve, NocedalWright, Hei, Yuan, Fan, Bastin}.  Bastin (trust_region.jl:484-503) reads a
   `δu_cache` that the reference allocates with `similar(u)` and never writes; the library uses the step just taken, which is
   what the retrospective scheme of the cited paper evaluates. */
enum { B200_TR_SIMPLE = 0, B200_TR_NLSOLVE = 1, B200_TR_NOCEDAL_WRIGHT = 2, B200_TR_HEI = 3, B200_TR_YUAN = 4, B200_TR_FAN = 5, B200_TR_BASTIN = 6 };
/* LEVENBERG_MARQUARDT (levenberg_marquardt.jl:36-61): DampedNewtonDescent with the Levenberg-Marquardt damping function
   (running maximum of diag(J'J), floor min_damping_D) wrapped in GeodesicAcceleration, with LevenbergMarquardtTrustRegion;
   concrete (dense) Jacobian; the damped system is solved in normal form, (J'J + lambda D'D) v = J'f */
enum { B200_DESCENT_NEWTON = 0, B200_DESCENT_PSEUDO_TRANSIENT = 1, B200_DESCENT_LEVENBERG_MARQUARDT = 2, B200_DESCENT_BROYDEN = 3 };
/* BROYDEN (NonlinearSolveQuasiNewton/src/broyden.jl:34-51; SURVEY.md §8f-4): the quasi-Newton family's Broyden() — NewtonDescent on a
   STORED INVERSE J^-1 (dense n x n, resident in HBM), rank-one good / bad Broyden update after every step, NoChangeInStateReset
   (reset_conditions.jl:18-88) re-initialising J^-1, ConvergenceFailure after max_resets.  The step routine is keyed on this field
   because the option struct is; in the reference it is its own algorithm type, not a descent. */
enum { B200_QN_INIT_IDENTITY = 0, B200_QN_INIT_TRUE_JACOBIAN = 1, B200_QN_INIT_LOW_RANK = 2 };
/* init_jacobian = Val(:identity) | Val(:true_jacobian) (needs linsolve = DENSE_LU); LOW_RANK = LimitedMemoryBroyden(; threshold)
   (lbroyden.jl:20-35, initialization.jl:139-298): J^-1 = alpha I + U V' with the last `qn_threshold` rank-one updates kept in two
   n x threshold arrays (circular), any n */
enum { B200_QN_UPDATE_GOOD_BROYDEN = 0, B200_QN_UPDATE_BAD_BROYDEN = 1, B200_QN_UPDATE_KLEMENT = 2 };
/* KLEMENT (klement.jl:30-49, 128-140): Klement() with its default init_jacobian = Val(:identity), i.e. a DIAGONAL approximate Jacobian
   (an n-vector, any n): du = -f ./ J, J += ((df - J du) ./ (J^2 du^2)) .* du .* J^2, IllConditionedJacobianReset (any zero on the diagonal) */
/* built-in preconditioners (LinearSolve `precs(A, p)`, large_systems.md:244-316): inverse of the 2x2 species blocks, or one
   geometric-multigrid V-cycle of the Brusselator Jacobian (the tutorial's AlgebraicMultigrid ruge_stuben / smoothed_aggregation) */
/* ILU0: incomplete LU with zero fill of the assembled sparse Jacobian (b200_ilu0_*), refactorised with every fresh Jacobian;
   needs linsolve = SPARSE_GMRES and works on any problem with a pattern (built-in or a callback's jac_prototype) */
/* AMG: one Ruge-Stueben algebraic-multigrid V-cycle of the assembled sparse Jacobian (b200_amg_*, default options): hierarchy
   rebuilt at the first fresh Jacobian after create / reinit, values refreshed on the device with every later one; needs
   linsolve = SPARSE_GMRES, any problem with a pattern */
/* SA_AMG: the same with smoothed aggregation (b200_amg_create_sa, default options): the whole rebuild runs on the device */
enum { B200_PRECOND_NONE = 0, B200_PRECOND_BLOCK_JACOBI_LEFT = 1, B200_PRECOND_BLOCK_JACOBI_RIGHT = 2,
       B200_PRECOND_MULTIGRID_LEFT = 3, B200_PRECOND_MULTIGRID_RIGHT = 4, B200_PRECOND_ILU0_LEFT = 5, B200_PRECOND_ILU0_RIGHT = 6,
       B200_PRECOND_AMG_LEFT = 7, B200_PRECOND_AMG_RIGHT = 8, B200_PRECOND_SA_AMG_LEFT = 9, B200_PRECOND_SA_AMG_RIGHT = 10 };
enum { B200_FORCING_NONE = 0, B200_FORCING_EW2 = 1 };
/* termination modes (public.jl:300-407, termination_conditions.jl:243-372); `du` = f(u).  The three AbsNorm modes keep
   their round-1 values; Norm / Rel / RelNorm / Abs / RelNormSafe / RelNormSafeBest follow */
enum { B200_TERM_ABS_NORM_SAFE_BEST = 0, B200_TERM_ABS_NORM = 1, B200_TERM_ABS_NORM_SAFE = 2, B200_TERM_NORM = 3, B200_TERM_REL = 4,
       B200_TERM_REL_NORM = 5, B200_TERM_ABS = 6, B200_TERM_REL_NORM_SAFE = 7, B200_TERM_REL_NORM_SAFE_BEST = 8 };
enum { B200_NORM_INF = 0, B200_NORM_L2 = 1 }; /* internalnorm: maximum(abs, .) (NonlinearProblem default) or norm(., 2) */
enum { B200_U0_REFERENCE = 0, B200_U0_PERTURBED_Z = 1 };
enum { B200_ORDER_NATURAL = 0, B200_ORDER_LARGEST_FIRST = 1 };

typedef struct b200_ctx b200_ctx;
typedef struct b200_problem b200_problem;
typedef struct b200_linop b200_linop;
typedef struct b200_gmres b200_gmres;
typedef struct b200_newton b200_newton;
typedef struct b200_sparse_jac b200_sparse_jac;
typedef struct b200_ensemble b200_ensemble;

/* host callbacks invoked between kernels (b1 plug-in point: an arbitrary Julia f!/jvp!/vjp! closure
 * through @cfunction).  Pointers are device pointers.  The library drains its own (non-blocking) streams before every
 * callback, so the arguments are ready on any stream; the callback's own device work must be enqueued on the ctx stream
 * (b200_ctx_stream) or be complete on return.  Return 0 on success. */
typedef int32_t (*b200_residual_cb)(void* user, const double* u, double* du);
typedef int32_t (*b200_jvp_cb)(void* user, const double* u, const double* v, double* Jv);
typedef int32_t (*b200_matvec_cb)(void* user, const double* x, double* y);
/* b3 plug-in point `jac = jac!` (jacobian.jl:241-243): fills the concrete Jacobian in place — J is the dense column-major
   n x n matrix (ld = n) for the dense path, or the nzval array of the CSC pattern given to b200_sparse_jac_create */
typedef int32_t (*b200_jac_cb)(void* user, const double* u, double* J);

/* ---------------------------------------------------------------- option / result structs */
typedef struct b200_gmres_opts {
  int32_t memory;     /* initial basis allocation; Krylov.jl `memory` (LinearSolve passes min(20,n)); grows on demand */
  int32_t restart;    /* 0 = never restart (KrylovJL_GMRES default gmres_restart=0); k>0 = GMRES(k) */
  int32_t itmax;      /* 0 => n (LinearSolve default maxiters = length(b)) */
  int32_t orth;       /* B200_ORTH_* ; MGS = Krylov.jl default (reorthogonalization=false) */
  int32_t warm_start; /* 0: x0 = 0 ; 1: x_inout holds the initial guess */
  int32_t engine;     /* B200_ENGINE_* */
  int32_t check_every;/* host polls the device status every this many Arnoldi iterations (multi-kernel engine); 0 => 8 (2 with a preconditioner) */
  int32_t block;      /* reserved, must be 0 (round 1 offered an L2-blocked Gram-Schmidt here: measured 2x slower than the
                         streaming kernels and removed) */
  double atol;
  double rtol;
} b200_gmres_opts;

typedef struct b200_gmres_stats {
  int32_t status;     /* B200_LS_* */
  int32_t iters;      /* Arnoldi iterations performed */
  int32_t nmatvec;    /* operator applications (iters + 1 if warm start) */
  int32_t restarts;
  double rnorm0;      /* ||b - A x0|| */
  double rnorm;       /* final residual-norm estimate from the Givens recurrence */
  double tol;         /* atol + rtol*rnorm0 */
  double bytes;       /* algorithmic HBM bytes moved by this solve (DESIGN.md accounting) */
} b200_gmres_stats;

typedef struct b200_newton_opts {
  double abstol;      /* <=0 => 3e-13 (common_defaults.jl:44-48) */
  double reltol;      /* <=0 => 3e-13 */
  int32_t maxiters;   /* <=0 => 1000 (solve.jl:142) */
  int32_t linsolve;   /* B200_LINSOLVE_* */
  int32_t jvp_mode;   /* B200_JVP_* */
  int32_t globalization;
  int32_t forcing;
  int32_t termination;
  int32_t store_trace;
  int32_t fused_step; /* reserved and ignored: the update u += du, the residual and both norms always run as the two fused kernels */
  b200_gmres_opts gmres; /* atol/rtol <= 0 => inherit the nonlinear abstol/reltol (solve.jl:203) */
  /* Eisenstat-Walker forcing (eisenstat_walker.jl:18-30) */
  double ew_eta0, ew_eta_max, ew_gamma, ew_alpha, ew_safeguard_threshold;
  int32_t ew_safeguard;
  int32_t max_shrink_times; /* trust_region.jl: 32 */
  /* trust region, RadiusUpdateSchemes.Simple defaults (trust_region.jl:320-384) ; 0 => default */
  double tr_step_threshold, tr_shrink_threshold, tr_expand_threshold, tr_shrink_factor, tr_expand_factor;
  double tr_max_trust_radius, tr_initial_trust_radius;
  /* BackTracking line search (globalization = LINESEARCH; solve.jl:249-273, 392-408; LineSearch.jl BackTracking, cubic
     interpolation): sufficient-decrease constant, step contraction bounds, max backtracks.  0 => 1e-4, 0.5, 0.1, 1000 */
  double ls_c1, ls_rho_hi, ls_rho_lo;
  int32_t ls_maxiters;
  int32_t precond; /* B200_PRECOND_*: built-in preconditioner handed to GMRES each step (LinearSolve `precs(A, p)`) */
  int32_t descent; /* B200_DESCENT_* */
  int32_t tr_scheme; /* B200_TR_*: RadiusUpdateSchemes (trust_region.jl:431-509); thresholds/factors of 0 take the scheme's defaults (:330-384) */
  double pt_alpha_initial; /* PseudoTransient(alpha_initial = 1e-3); 0 => 1e-3 */
  double maxtime;          /* seconds of accumulated step time after which the solve stops with MaxTime (NonlinearSolveBase/src/solve.jl:847-855); <= 0 => none */
  int32_t term_norm;       /* B200_NORM_*: the termination mode's internalnorm */
  int32_t term_max_stalled_steps; /* Safe modes: window of the step-norm stall test; 0 => 32 (the solver default's value), < 0 => test disabled */
  /* LevenbergMarquardt(; damping_initial = 1, damping_increase_factor = 2, damping_decrease_factor = 3, finite_diff_step_geodesic
     = 0.1, α_geodesic = 0.75, b_uphill = 1, min_damping_D = 1e-8, disable_geodesic = Val(false)); 0 => the default */
  double lm_damping_initial, lm_damping_increase, lm_damping_decrease, lm_finite_diff_step, lm_alpha_geodesic, lm_b_uphill, lm_min_damping_D;
  int32_t lm_disable_geodesic;
  int32_t reserved0;
  /* Broyden(; max_resets = 100, reset_tolerance = eps^(3/4), init_jacobian = Val(:identity), alpha = nothing, update_rule =
     Val(:good_broyden)); qn_alpha <= 0 => 2 ||f|| / max(||u||, 1) (1 when ||f|| < 1e-5), the identity is scaled by it before
     inversion */
  int32_t qn_init_jacobian, qn_update_rule, qn_max_resets, qn_threshold; /* qn_threshold: LOW_RANK only; 0 => 10 */
  double qn_reset_tolerance, qn_alpha;
} b200_newton_opts;

typedef struct b200_newton_result {
  int32_t retcode;    /* B200_RC_* */
  int32_t nsteps;     /* NLStats.nsteps */
  int32_t nf;         /* NLStats.nf   */
  int32_t njacs;      /* NLStats.njacs */
  int32_t nfactors;   /* NLStats.nfactors */
  int32_t nsolve;     /* NLStats.nsolve */
  int32_t njvp;       /* total Arnoldi operator applications */
  int32_t ntrace;
  double resid_inf;   /* ||f(u)||_inf at the returned u */
  double bytes;       /* algorithmic HBM bytes (DESIGN.md accounting) */
} b200_newton_result;

typedef struct b200_trace_rec {
  int32_t iter;
  int32_t lin_iters;
  int32_t lin_status;
  int32_t accepted;   /* trust region: step accepted */
  double fnorm_inf;   /* ||f(u_iter)||_inf */
  double step_norm2;  /* ||u_iter - u_{iter-1}||_2 */
  double lin_rnorm;
  double trust_radius;
} b200_trace_rec;

/* ---------------------------------------------------------------- context, memory, events */
int32_t b200_version(void);
int32_t b200_device_count(int32_t* count);
/* stream: an existing cudaStream_t to enqueue on (e.g. torch's current stream), or NULL to create one */
int32_t b200_ctx_create(int32_t device, void* stream, b200_ctx** ctx);
int32_t b200_ctx_destroy(b200_ctx* ctx);
int32_t b200_ctx_sync(b200_ctx* ctx);
void* b200_ctx_stream(b200_ctx* ctx);
const char* b200_last_error(b200_ctx* ctx);
/* number of kernels this library launched on ctx since creation (bench.py's gpu_launches) */
int32_t b200_ctx_kernel_launches(b200_ctx* ctx, int64_t* count);
int32_t b200_ctx_sm_count(b200_ctx* ctx, int32_t* count);
/* per-kernel-family device timing with CUDA events on the ctx stream (bench.py's live roofline measurement);
 * bytes = the algorithmic HBM bytes of the timed launches (DESIGN.md accounting). */
enum { B200_KID_JVP = 0, B200_KID_MULTIDOT = 1, B200_KID_UPDATE = 2, B200_KID_MGS = 3, B200_KID_NORMALIZE = 4,
       B200_KID_RESIDUAL = 5, B200_KID_GIVENS = 6, B200_KID_RESIDENT = 7, B200_KID_LU_PANEL = 8, B200_KID_LU_GEMM = 9,
       B200_KID_LU_OTHER = 10, B200_KID_SPARSE = 11, B200_KID_COUNT = 12 };
int32_t b200_ctx_profile_enable(b200_ctx* ctx, int32_t on);
int32_t b200_ctx_profile_reset(b200_ctx* ctx);
int32_t b200_ctx_profile_get(b200_ctx* ctx, int32_t kernel_id, double* ms_host, double* bytes_host, int64_t* launches_host);

int32_t b200_malloc(b200_ctx* ctx, size_t bytes, void** dptr);
int32_t b200_free(b200_ctx* ctx, void* dptr);
int32_t b200_host_alloc(b200_ctx* ctx, size_t bytes, void** hptr); /* pinned */
int32_t b200_host_free(b200_ctx* ctx, void* hptr);
int32_t b200_memcpy_h2d(b200_ctx* ctx, void* dst, const void* src_host, size_t bytes);
int32_t b200_memcpy_d2h(b200_ctx* ctx, void* dst_host, const void* src, size_t bytes);
int32_t b200_memcpy_d2d(b200_ctx* ctx, void* dst, const void* src, size_t bytes);
int32_t b200_memset(b200_ctx* ctx, void* dst, int32_t byte, size_t bytes);
int32_t b200_flush_l2(b200_ctx* ctx); /* overwrite a >L2-sized scratch buffer (bench hygiene) */

/* ---------------------------------------------------------------- vector ops (b5: what L2-L4 touch on a device array) */
int32_t b200_fill(b200_ctx* ctx, int64_t n, double a, double* x);
int32_t b200_copy(b200_ctx* ctx, int64_t n, const double* x, double* y);
int32_t b200_scal(b200_ctx* ctx, int64_t n, double a, double* x);
int32_t b200_axpy(b200_ctx* ctx, int64_t n, double a, const double* x, double* y);             /* y += a x */
int32_t b200_axpby(b200_ctx* ctx, int64_t n, double a, const double* x, double b, double* y);  /* y = a x + b y */
int32_t b200_mul(b200_ctx* ctx, int64_t n, const double* x, const double* y, double* z);       /* z = x .* y */
int32_t b200_dot(b200_ctx* ctx, int64_t n, const double* x, const double* y, double* out_host);
int32_t b200_nrm2(b200_ctx* ctx, int64_t n, const double* x, double* out_host);
int32_t b200_norminf(b200_ctx* ctx, int64_t n, const double* x, double* out_host);             /* maximum(abs, x) */
int32_t b200_diffnrm2(b200_ctx* ctx, int64_t n, const double* x, const double* y, double* out_host); /* ||x-y||_2 */
int32_t b200_extrema(b200_ctx* ctx, int64_t n, const double* x, double* min_host, double* max_host);
int32_t b200_equal(b200_ctx* ctx, int64_t n, const double* x, const double* y, int32_t* equal_host);

/* ---------------------------------------------------------------- problems (a1, a2) */
int32_t b200_problem_create_bruss2d(b200_ctx* ctx, int32_t N, double A, double B, double alpha, b200_problem** prob);
int32_t b200_problem_create_bruss3d(b200_ctx* ctx, int32_t N, double A, double B, double alpha, b200_problem** prob);
int32_t b200_problem_create_quadratic(b200_ctx* ctx, int64_t n, double p, b200_problem** prob);          /* f = u.^2 .- p */
int32_t b200_problem_create_tridiag_quad(b200_ctx* ctx, int64_t n, const double* p_dev, b200_problem** prob); /* rootfind_tests__item20.jl */
int32_t b200_problem_create_callback(b200_ctx* ctx, int64_t n, b200_residual_cb f, b200_jvp_cb jvp, b200_jvp_cb vjp,
                                     void* user, b200_problem** prob);
/* user Jacobian fills (either may be NULL): used by b200_dense_jac_fill / b200_sparse_jac_fill instead of JVP sweeps */
int32_t b200_problem_set_jac(b200_problem* prob, b200_jac_cb jac_dense, b200_jac_cb jac_nzval);
/* `jac_prototype = J0::SparseMatrixCSC` for problems without a built-in pattern (jacobian.jl:119-125): the structure that
   b200_pattern(_nnz) — and therefore the sparse path of the Newton driver — report for this problem.  Copied. */
int32_t b200_problem_set_jac_prototype(b200_problem* prob, const int64_t* colptr, const int64_t* rowval, int32_t index_base);
int32_t b200_problem_destroy(b200_problem* prob);
int32_t b200_problem_n(b200_problem* prob, int64_t* n);
int32_t b200_problem_set_AB(b200_problem* prob, double A, double B);     /* remake(prob; p = ...) */
int32_t b200_problem_u0(b200_problem* prob, int32_t mode, double* u);    /* reference initial condition */
int32_t b200_residual(b200_problem* prob, const double* u, double* du);
int32_t b200_jvp(b200_problem* prob, const double* u, const double* v, double* Jv);                      /* exact tangent */
int32_t b200_residual_jvp(b200_problem* prob, const double* u, const double* v, double* du, double* Jv); /* one halo load */
int32_t b200_jvp_fd(b200_problem* prob, const double* u, const double* v, double* Jv);                   /* (f(u+eps v)-f(u))/eps, fused */
int32_t b200_vjp(b200_problem* prob, const double* u, const double* w, double* JTw);

/* ---------------------------------------------------------------- linear operators + GMRES (a3) */
int32_t b200_linop_from_problem(b200_problem* prob, const double* u, int32_t jvp_mode, b200_linop** op);
int32_t b200_linop_from_csc(b200_ctx* ctx, int64_t n, const int64_t* colptr_dev, const int64_t* rowval_dev,
                            const double* nzval_dev, int32_t index_base, b200_linop** op);
int32_t b200_linop_from_dense(b200_ctx* ctx, int64_t n, const double* A_dev, int64_t ld, b200_linop** op);
int32_t b200_linop_from_callback(b200_ctx* ctx, int64_t n, b200_matvec_cb mv, void* user, b200_linop** op);
int32_t b200_linop_apply(b200_linop* op, const double* x, double* y);
/* A + shift I  (dampen_jacobian!!(cache, J::AbstractSciMLOperator, D) = J + D, descent/damped_newton.jl) */
int32_t b200_linop_set_shift(b200_linop* op, double shift);
int32_t b200_linop_destroy(b200_linop* op);

void b200_gmres_opts_default(b200_gmres_opts* opts);
int32_t b200_gmres_create(b200_ctx* ctx, int64_t n, const b200_gmres_opts* opts, b200_gmres** gm);
int32_t b200_gmres_destroy(b200_gmres* gm);
int32_t b200_gmres_set_tolerances(b200_gmres* gm, double atol, double rtol); /* LinearSolve.update_tolerances! */
/* Preconditioning (SURVEY.md §8 b4 / f2: `KrylovJL_GMRES(precs = (A, p) -> (Pl, Pr))`, test/Core/core_tests__item21.jl;
 * Krylov.jl gmres!(…; M = Pl, N = Pr, ldiv = false)): each operator APPLIES the inverse, y = M^-1 x.  Left: the Krylov
 * method runs on M^-1 A x = M^-1 b and its stopping test sees the preconditioned residual; right: A N^-1 y = b, x = N^-1 y.
 * NULL clears a side.  The operators are borrowed (caller keeps them alive until the solve returns). */
int32_t b200_gmres_set_precond(b200_gmres* gm, b200_linop* left_inv, b200_linop* right_inv);
/* Built-in block-Jacobi preconditioner of the Brusselator Jacobian at u: inverse of the 2x2 species blocks on the diagonal
 * (large_systems.md:244-316 uses an incomplete LU / multigrid of the same matrix through `precs`). */
int32_t b200_linop_block_jacobi(b200_problem* prob, const double* u, b200_linop** out);
/* Built-in preconditioner by kind (B200_PRECOND_*, the LEFT / RIGHT values of a family name the same operator): block-Jacobi
 * or one multigrid V-cycle of the Brusselator Jacobian at u — coarsening by the prime factors of N down to one cell,
 * damped block-Jacobi smoothing (2 pre + 2 post sweeps), trilinear / full-weighting transfers for factor 2 and aggregation
 * for odd factors, rediscretised coarse operators, exact 2x2 solve on the last level.  The operator applies M^-1. */
int32_t b200_linop_precond(b200_problem* prob, const double* u, int32_t kind, b200_linop** out);
int32_t b200_gmres_solve(b200_gmres* gm, b200_linop* op, const double* b, double* x_inout, b200_gmres_stats* stats_host);

/* ---------------------------------------------------------------- dense fallback (a5) */
int32_t b200_dense_jac_fill(b200_problem* prob, const double* u, double* J, int64_t ld); /* column-major n x n */
int32_t b200_getrf(b200_ctx* ctx, int64_t n, double* A, int64_t ld, int64_t* ipiv_dev, int32_t* info_host); /* LAPACK getrf semantics, 1-based ipiv */
int32_t b200_getrs(b200_ctx* ctx, int64_t n, int64_t nrhs, const double* A, int64_t ld, const int64_t* ipiv_dev,
                   double* B, int64_t ldb);
int32_t b200_gemv(b200_ctx* ctx, int32_t trans, int64_t m, int64_t n, const double* A, int64_t ld, const double* x, double* y);

/* ---------------------------------------------------------------- sparse fallback (a6) */
int32_t b200_pattern_nnz(b200_problem* prob, int64_t* nnz);
int32_t b200_pattern(b200_problem* prob, int32_t index_base, int64_t* colptr_host, int64_t* rowval_host); /* CSC, sorted rows */
int32_t b200_coloring_column(int64_t n, const int64_t* colptr_host, const int64_t* rowval_host, int32_t index_base,
                             int32_t order, int64_t* colors_host /* 1-based */, int64_t* ncolors_host);
int32_t b200_sparse_jac_create(b200_problem* prob, const int64_t* colptr_host, const int64_t* rowval_host, int32_t index_base,
                               const int64_t* colors_host, int64_t ncolors, b200_sparse_jac** sj);
int32_t b200_sparse_jac_destroy(b200_sparse_jac* sj);
int32_t b200_sparse_jac_fill(b200_sparse_jac* sj, const double* u, double* nzval_dev); /* ncolors seeded JVP sweeps + scatter */
int32_t b200_sparse_jac_linop(b200_sparse_jac* sj, const double* nzval_dev, b200_linop** op);
int32_t b200_spmv(b200_sparse_jac* sj, const double* nzval_dev, const double* x, double* y);   /* y = J x  */
int32_t b200_spmv_t(b200_sparse_jac* sj, const double* nzval_dev, const double* x, double* y); /* y = J' x */

/* ---------------------------------------------------------------- sparse direct solve (a6; small 2D / 3D grids)
 * Reverse Cuthill-McKee ordering of the pattern (host, once), then LAPACK-gbtrf-style banded LU with partial pivoting and
 * the two banded triangular solves on the device.  Memory n * (2 kl + ku + 1) doubles: B200_ERR_NOMEM when the band does not
 * fit (3D N = 100: use GMRES on the assembled matrix, as the reference's own GPU test does). */
typedef struct b200_sparse_lu b200_sparse_lu;
int32_t b200_sparse_lu_create(b200_ctx* ctx, int64_t n, const int64_t* colptr_host, const int64_t* rowval_host, int32_t index_base,
                              b200_sparse_lu** lu);
int32_t b200_sparse_lu_destroy(b200_sparse_lu* lu);
int32_t b200_sparse_lu_bandwidth(b200_sparse_lu* lu, int64_t* kl_host, int64_t* ku_host);
int32_t b200_sparse_lu_factor(b200_sparse_lu* lu, const double* nzval_dev, int32_t* info_host);   /* info > 0: zero pivot at that column (1-based) */
int32_t b200_sparse_lu_solve(b200_sparse_lu* lu, const double* b_dev, double* x_dev);            /* x = A^-1 b (x may alias b) */

/* ---------------------------------------------------------------- ILU(0) preconditioner of an assembled sparse matrix
 * Incomplete LU with the sparsity pattern of A (no fill, no pivoting): the first `precs` of large_systems.md:244-316.
 * Symbolic phase on the host, once per pattern: CSR view with int32 indices (n, nnz < 2^31), diagonal positions, level sets
 * of the strictly lower and strictly upper patterns.  Factorisation and solve run on the device, level by level in one
 * cooperative launch each; results are bit-reproducible.  A row without a structural diagonal fails create with
 * B200_ERR_INVALID (the message names the row). */
typedef struct b200_ilu0 b200_ilu0;
int32_t b200_ilu0_create(b200_ctx* ctx, int64_t n, const int64_t* colptr_host, const int64_t* rowval_host, int32_t index_base, b200_ilu0** ilu);
int32_t b200_ilu0_destroy(b200_ilu0* ilu);
int32_t b200_ilu0_levels(b200_ilu0* ilu, int32_t* lower_host, int32_t* upper_host);   /* level counts of the forward / backward sweep */
int32_t b200_ilu0_factor(b200_ilu0* ilu, const double* nzval_dev, int32_t* info_host);  /* info > 0: zero or non-finite pivot u_ii at that row (1-based) */
int32_t b200_ilu0_solve(b200_ilu0* ilu, const double* b_dev, double* x_dev);           /* x = U^-1 L^-1 b, L unit lower (x may alias b) */
/* the packed factors in the caller's CSC order: L strictly below the diagonal (unit diagonal implied), U on and above it */
int32_t b200_ilu0_export(b200_ilu0* ilu, double* nzval_out_dev);
/* an operator applying U^-1 L^-1, for b200_gmres_set_precond; it borrows the handle (destroy the operator first) */
int32_t b200_ilu0_linop(b200_ilu0* ilu, b200_linop** op);

/* ---------------------------------------------------------------- algebraic multigrid preconditioner of an assembled sparse matrix
 * Classical Ruge-Stueben AMG (the second `precs` of large_systems.md:244-316, with Jacobi smoothing; DESIGN.md §4h states the
 * rules): classical strength (theta), the deterministic first-pass C/F splitting, direct interpolation, Galerkin coarse operators
 * R A P with R = P', an explicit dense inverse of the coarsest level (at most 4096 unknowns).  The pattern (int32 CSR indices,
 * n and every level's nnz < 2^31) is fixed at create.
 *   setup(rebuild = 1): chooses each level's splitting on the host from its values, builds every pattern and value on the device
 *                       (the coarse values come down for the next splitting), then runs the device refresh;  setup(rebuild = 0): the splitting and patterns stay, the device recomputes every
 *                       value (bit-reproducible; equal bits to a rebuild at the same values).
 *   solve: one V(presweeps, postsweeps) cycle with damped Jacobi from x = 0, replayed as one CUDA graph; a fixed linear operator.
 * info > 0: the 1-based level whose diagonal (or interpolation denominator) is zero or not finite, or whose dense LU met a zero
 * pivot (coarsest level).  A hierarchy that ends above 4096 unknowns fails setup with B200_ERR_UNSUPPORTED. */
typedef struct b200_amg b200_amg;
typedef struct b200_amg_opts {
  double theta;        /* strength threshold: 0.25 */
  double omega;        /* Jacobi damping: 2/3 */
  int32_t presweeps;   /* 1 */
  int32_t postsweeps;  /* 1 */
  int32_t max_levels;  /* 10 (the finest level counts) */
  int32_t max_coarse;  /* 10: a level of at most this many unknowns is the coarsest */
} b200_amg_opts;
enum { B200_AMG_EXPORT_A = 0, B200_AMG_EXPORT_P = 1, B200_AMG_EXPORT_T = 2 /* smoothed aggregation only */ };
void b200_amg_opts_default(b200_amg_opts* opts);
/* opts NULL: the defaults.  A row without a structural diagonal fails with B200_ERR_INVALID (the message names the row). */
int32_t b200_amg_create(b200_ctx* ctx, int64_t n, const int64_t* colptr_host, const int64_t* rowval_host, int32_t index_base,
                        const b200_amg_opts* opts, b200_amg** amg);
int32_t b200_amg_destroy(b200_amg* amg);
int32_t b200_amg_setup(b200_amg* amg, const double* nzval_dev, int32_t rebuild, int32_t* info_host);
int32_t b200_amg_solve(b200_amg* amg, const double* b_dev, double* x_dev);  /* x = M^-1 b (x may alias b) */
/* number of levels; the unknowns and nonzeros of the first `cap` of them */
int32_t b200_amg_levels(b200_amg* amg, int32_t* nlev_host, int64_t* n_per_level_host, int64_t* nnz_per_level_host, int32_t cap);
/* the CSR (0-based, int32 indices, columns ascending) of A_level, of P_level or (smoothed aggregation) of the tentative
   prolongator T_level, whose row i holds one entry in the column of i's aggregate or none (n_level x n_level+1; P and T not on
   the coarsest level); rowptr holds n_level + 1 entries, col / val rowptr[n_level]; with col and val NULL only rowptr is written */
int32_t b200_amg_export(b200_amg* amg, int32_t level, int32_t what, int32_t* rowptr_host, int32_t* col_host, double* val_host);
/* an operator applying one V-cycle, for b200_gmres_set_precond; it borrows the handle (destroy the operator first) */
int32_t b200_amg_linop(b200_amg* amg, b200_linop** op);
/* Smoothed-aggregation AMG (AlgebraicMultigrid.jl's `smoothed_aggregation`, one candidate; DESIGN.md §4i states the rules):
 * symmetric strength |a_ij| >= theta sqrt(|a_ii| |a_jj|), aggregates grown from a distance-2 maximal independent set, the
 * tentative prolongator T (unit columns, b_next = the aggregates' norms of b, b = 1 on the finest level) and
 * P = T - (smooth_omega / rho) D^-1 A T with rho the Gershgorin bound of D^-1 A.  The handle is a b200_amg: setup, solve, levels,
 * export and linop work as above, and setup(rebuild = 1) runs on the device with no host pass over the matrix. */
typedef struct b200_sa_opts {
  double theta;          /* strength threshold: 0.08 */
  double omega;          /* Jacobi damping of the cycle: 2/3 */
  int32_t presweeps;     /* 1 */
  int32_t postsweeps;    /* 1 */
  int32_t max_levels;    /* 10 (the finest level counts) */
  int32_t max_coarse;    /* 10: a level of at most this many unknowns is the coarsest */
  double smooth_omega;   /* prolongator smoothing weight omega_P: 4/3 */
} b200_sa_opts;
void b200_sa_opts_default(b200_sa_opts* opts);
int32_t b200_amg_create_sa(b200_ctx* ctx, int64_t n, const int64_t* colptr_host, const int64_t* rowval_host, int32_t index_base,
                           const b200_sa_opts* opts, b200_amg** amg);
/* the level-0 C/F splitting alone, on the host (no device): cf_out[i] = 1 for a C point, 0 for an F point */
int32_t b200_amg_split(int64_t n, const int64_t* colptr_host, const int64_t* rowval_host, const double* nzval_host, int32_t index_base,
                       double theta, int32_t* cf_out_host, int64_t* ncoarse_host);

/* ---------------------------------------------------------------- Newton driver (a4, a7, a8, a9) */
void b200_newton_opts_default(b200_newton_opts* opts);
int32_t b200_newton_create(b200_problem* prob, const b200_newton_opts* opts, b200_newton** nw);
int32_t b200_newton_destroy(b200_newton* nw);
int32_t b200_newton_reinit(b200_newton* nw, const double* u0_dev);            /* reinit!(cache, u0) */
int32_t b200_newton_step(b200_newton* nw, int32_t* terminated_host);           /* step!(cache) */
int32_t b200_newton_solve(b200_newton* nw, b200_newton_result* result_host);   /* solve!(cache) */
int32_t b200_newton_result_get(b200_newton* nw, b200_newton_result* result_host);
int32_t b200_newton_u(b200_newton* nw, double** u_dev);
int32_t b200_newton_fu(b200_newton* nw, double** fu_dev);
int32_t b200_newton_trace(b200_newton* nw, b200_trace_rec* recs_host, int32_t cap, int32_t* count_host);
/* whole-solve convenience with HOST buffers (H2D of u0, solve, D2H of u and resid): the e2e call */
int32_t b200_newton_solve_host(b200_newton* nw, const double* u0_host, double* u_host, double* resid_host,
                               b200_newton_result* result_host);

/* ---------------------------------------------------------------- ensemble (a11): K independent 2D Brusselators
 * Trajectories are matrix-free NewtonRaphson solves with GMRES.  The preconditioner may be none, block-Jacobi or multigrid
 * (either side); ILU0 and AMG need the assembled sparse Jacobian and are refused with B200_ERR_INVALID.  For N <= 32 one kernel
 * solves the whole batch, one CTA per trajectory, with the multigrid V-cycle in shared memory; block-Jacobi, N > 32 and the
 * option sets that kernel does not cover run the single-system driver, one trajectory after another. */
typedef struct b200_ens_result {
  int32_t nprob;
  int32_t nsuccess;
  int32_t max_nsteps;
  int32_t reserved;
  int64_t total_nsteps;
  int64_t total_njvp;
  double worst_resid_inf;
} b200_ens_result;
int32_t b200_ens_create(b200_ctx* ctx, int32_t N, int32_t nprob_local, double alpha, const b200_newton_opts* opts, b200_ensemble** ens);
int32_t b200_ens_destroy(b200_ensemble* ens);
/* u0: nprob x n (problem-major, each problem a contiguous (N,N,2) block); A,B: per-problem parameters */
int32_t b200_ens_solve(b200_ensemble* ens, const double* u0_dev, const double* A_dev, const double* B_dev, double* u_out_dev,
                       double* resid_inf_dev, int32_t* retcodes_dev, int32_t* nsteps_dev, int32_t* njvp_dev,
                       b200_ens_result* result_host);
/* y_m = M_m^-1 x_m for every trajectory m of a batched multigrid ensemble: M_m is the V-cycle at iterate u_m with parameter
   A_m, applied by the solve kernel's own device routine (u, x, y: nprob x n like u0; A: nprob).  B200_ERR_INVALID for any
   other ensemble. */
int32_t b200_ens_precond_apply(b200_ensemble* ens, const double* u_dev, const double* A_dev, const double* x_dev, double* y_dev);
/* resident CTAs per SM of the batched solve kernel for this ensemble's options (the occupancy query that sizes its grid);
   0 when its trajectories take the single-system driver */
int32_t b200_ens_ctas_per_sm(b200_ensemble* ens, int32_t* ctas_per_sm);

/* ---------------------------------------------------------------- collective step of the ensemble path (SURVEY.md §8b, §8e)
 * The ensemble shards by contiguous trajectory blocks, rank r owning [r K/R, (r+1) K/R): no collective on the data path.
 * After the solve: ONE all-gather of the solutions (EnsembleSolution.u in trajectory order on every rank) and one
 * all-reduce of the status counters, NCCL over NVLink / NVSwitch, enqueued on the context's stream (ordered after the solve
 * kernel, no host synchronisation in between).  Replaces what SciMLBase's `__solve(::EnsembleProblem, ...)` does when it
 * collects the per-trajectory solutions (test/PolyAlgorithms/core_tests__item6.jl:14-20); a host without torch.distributed
 * (the Julia glue, tests/abi_c) runs BASELINE config 5 on 8 GPUs through these calls.  NCCL is bound at run time
 * (dlopen of libnccl.so.2; B200_ERR_UNSUPPORTED when it cannot be loaded). */
typedef struct b200_comm b200_comm;
#define B200_NCCL_UNIQUE_ID_BYTES 128
int32_t b200_nccl_version(int32_t* version_host);
/* one process per GPU: rank 0 creates the id, the host language ships the 128 bytes to the other ranks (MPI / sockets /
   a file), every rank calls b200_nccl_init with the same id */
int32_t b200_nccl_unique_id(void* id128_host);
int32_t b200_nccl_init(b200_ctx* ctx, int32_t nranks, int32_t rank, const void* unique_id128_host, b200_comm** comm);
/* single process driving ndev devices (ncclCommInitAll): comms[i] belongs to ctxs[i]; wrap the per-device collective calls
   of one step in b200_nccl_group_start / _end */
int32_t b200_nccl_init_all(b200_ctx* const* ctxs, int32_t ndev, b200_comm** comms);
int32_t b200_nccl_group_start(void);
int32_t b200_nccl_group_end(void);
int32_t b200_nccl_destroy(b200_comm* comm);
/* u_all[r * count_local + i] = u_local[i] of rank r (count_local doubles per rank, equal on all ranks) */
int32_t b200_ens_allgather(b200_comm* comm, const double* u_local_dev, int64_t count_local, double* u_all_dev);
/* sums of nprob / nsuccess / total_nsteps / total_njvp, maxima of max_nsteps / worst_resid_inf over the ranks;
   _begin enqueues (usable inside a group), _finish synchronises the stream and fills the struct */
int32_t b200_ens_allreduce_stats_begin(b200_comm* comm, const b200_ens_result* local_host);
int32_t b200_ens_allreduce_stats_finish(b200_comm* comm, b200_ens_result* global_host);
int32_t b200_ens_allreduce_stats(b200_comm* comm, const b200_ens_result* local_host, b200_ens_result* global_host);

#ifdef __cplusplus
}
#endif
#endif /* B200NEWTON_H */
