// newton.cu — the first-order nonlinear driver on the device (SURVEY.md §8a rows a4, a7, a8, a9; kernels K5/K6).
//
// Mirrors GeneralizedFirstOrderAlgorithm: __init (lib/NonlinearSolveFirstOrder/src/solve.jl:140-301), step! (:325-465),
// the driver loop (lib/NonlinearSolveBase/src/solve.jl:360-387, 835-858), NewtonDescent (descent/newton.jl:97-141),
// Dogleg (descent/dogleg.jl:86-151), GenericTrustRegionScheme / RadiusUpdateSchemes.Simple (trust_region.jl:204-258,
// 320-384, 396-430, 511-513), EisenstatWalkerForcing2 (eisenstat_walker.jl:42-87) and the default termination mode
// AbsNormSafeBestTerminationMode (termination_conditions.jl:134-179, 243-336, 376-393, 414-453).
//
// All n-vectors stay in HBM for the whole solve; per step the host reads back one small record of scalars
// (||f||_inf, ||du||_2^2) produced by the epilogues of the update / residual kernels, and takes the (scalar) control
// decisions of the reference on the host.
#include "common.cuh"
#include <math.h>
#include <algorithm>
#include <chrono>
#include <initializer_list>

namespace {
struct TermCache {  // NonlinearTerminationModeCache (termination_conditions.jl:60-98)
  int mode;
  int norm_kind;        // B200_NORM_*
  int max_stalled;      // window of the step-norm stall test (0: disabled)
  double abstol, reltol, best, initial, u0_norm;
  int nsteps;
  int retcode;
  double obj_trace[100];
  double step_trace[128];
};
// what the modes read of (du = f(u), u): filled on demand by term_quantities()
struct TermQuant {
  double f_inf, f_norm, sum_norm, rel_viol;  // ||f||_inf ; internalnorm(f) ; internalnorm(f + u) ; #{ |f_i| > reltol |u_i + f_i| }
};
}  // namespace

struct b200_newton {
  b200_ctx* ctx;
  b200_problem* prob;
  b200_newton_opts o;
  int64_t n;
  double abstol, reltol;
  int maxiters;
  std::vector<void*> allocs;  // every device buffer of the driver (dev_alloc), freed by b200_newton_destroy
  double *u, *fu, *du, *xlin, *best_u;
  double *u_trial, *fu_trial, *Jdu, *JTfu, *du_c, *c1, *c2;
  b200_gmres* gm;
  b200_linop op;
  b200_linop prec;  // built-in preconditioner (opts.precond), re-pointed at the current iterate every step
  b200_mg* mg;      // multigrid hierarchy when opts.precond is MULTIGRID_*
  // dense
  double* Jdense;
  int64_t* ipiv;
  double* qr_work;    // pivoted-QR rescue of a singular LU (allocated on first use)
  int32_t* qr_jpvt;
  // sparse
  b200_sparse_jac* sj;
  double* nzval;
  b200_sparse_lu* slu;  // LINSOLVE_SPARSE_LU: band factorisation of the assembled Jacobian
  b200_ilu0* ilu;       // PRECOND_ILU0_*: incomplete LU of the assembled Jacobian, refactorised with every fresh J
  int32_t ilu_info;     // its last factorisation: 0, or the 1-based row of a zero / non-finite pivot
  b200_amg* amg;        // PRECOND_AMG_* / PRECOND_SA_AMG_*: Ruge-Stueben or smoothed-aggregation hierarchy of the assembled Jacobian
  int32_t amg_info;     // its last setup: 0, or the 1-based level of a zero diagonal / pivot
  int32_t amg_built;    // a hierarchy exists for this solve: later fresh Jacobians refresh its values (reset by reinit)
  // LevenbergMarquardt: J'J + lambda D'D (factored in place), the running diagonal D'D, velocity / acceleration, previous velocity, J' f
  double *lmA, *lm_dtd, *lm_v, *lm_a, *lm_vold, *lm_rhs;
  double lm_lambda, lm_lambda_factor, lm_norm_v_old, lm_loss_old;
  // Broyden family: the previous residual of the update rule (Klement's fu_cache) and of the reset test; the stored inverse
  // (n x n, dense form only), J^-1 df, the rule's row vector w and rank-one column c; Klement's diagonal J (not inverted)
  double *qn_dfu, *qn_dfu_reset, *qn_Jinv, *qn_Jdfu, *qn_w, *qn_c, *kl_J;
  int qn_since_du, qn_since_dfu, qn_nresets;  // Broyden: NoChangeInStateReset counters, resets so far
  double *lr_U, *lr_V, *lr_c;                // LimitedMemoryBroyden: J^-1 = lr_alpha I + U V' (n x lr_m each, circular), coefficient scratch
  int lr_m, lr_idx;
  double lr_alpha;
  // state
  TermCache tc;
  b200_newton_result res;
  std::vector<b200_trace_rec> trace;
  int retcode, force_stop, make_new_jacobian, nsteps, have_factor, initialised;
  TrParams trp;
  double trust_region, max_tr;
  int shrink_counter;
  double eta, rnorm, rnorm_prev;
  double tp1, tp2, tp3, tp4;      // radius-update scheme parameters (get_parameters, trust_region.jl:372-379)
  double alpha_inv, pt_res_norm;  // PseudoTransient: 1/alpha and the residual 2-norm of the previous step (SER)
  double fnorm_inf;  // ||f(u)||_inf of the current iterate
  double total_time; // accumulated wall time of the steps (maxtime)
  double bytes;
};

namespace {
// ||x||_2 on the host (synchronising)
int32_t h_nrm2(b200_newton* nw, const double* x, double* out) { return b200_nrm2(nw->ctx, nw->n, x, out); }
int32_t h_dot(b200_newton* nw, const double* x, const double* y, double* out) { return b200_dot(nw->ctx, nw->n, x, y, out); }

bool term_is_safe(int mode) {
  return mode == B200_TERM_ABS_NORM_SAFE_BEST || mode == B200_TERM_ABS_NORM_SAFE || mode == B200_TERM_REL_NORM_SAFE || mode == B200_TERM_REL_NORM_SAFE_BEST;
}
bool term_is_best(int mode) { return mode == B200_TERM_ABS_NORM_SAFE_BEST || mode == B200_TERM_REL_NORM_SAFE_BEST; }
bool term_is_rel(int mode) { return mode == B200_TERM_REL_NORM_SAFE || mode == B200_TERM_REL_NORM_SAFE_BEST; }

// the reductions over (fu, u) a mode needs beyond ||fu||_inf (which the residual kernel's epilogue already produced)
int32_t term_quantities(b200_newton* nw, const double* fu, const double* u, double f_inf, TermQuant* q) {
  b200_ctx* ctx = nw->ctx;
  const int64_t n = nw->n;
  const int mode = nw->tc.mode;
  const bool l2 = nw->tc.norm_kind == B200_NORM_L2;
  q->f_inf = f_inf; q->f_norm = f_inf; q->sum_norm = 0.0; q->rel_viol = 0.0;
  const bool need_sum = mode == B200_TERM_NORM || mode == B200_TERM_REL_NORM || term_is_rel(mode);
  const bool need_viol = mode == B200_TERM_REL;
  const bool need_f2 = l2 && mode != B200_TERM_ABS && mode != B200_TERM_REL;
  if (!need_sum && !need_viol && !need_f2) return B200_OK;
  if (need_f2) B200_TRY(b200i_reduce_sum_dev(ctx, n, fu, nullptr, RED_SUMSQ, ctx->d_scalars + 8));
  if (need_sum) B200_TRY(b200i_reduce_sum_dev(ctx, n, fu, u, l2 ? RED_SUMSQ2 : RED_MAXABS2, ctx->d_scalars + 9));
  if (need_viol) B200_TRY(b200i_reduce_sum_dev(ctx, n, fu, u, RED_RELVIOL, ctx->d_scalars + 10, nw->tc.reltol));
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->h_scalars + 8, ctx->d_scalars + 8, sizeof(double) * 3, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (need_f2) q->f_norm = sqrt(ctx->h_scalars[8]);
  if (need_sum) q->sum_norm = l2 ? sqrt(ctx->h_scalars[9]) : ctx->h_scalars[9];
  if (need_viol) q->rel_viol = ctx->h_scalars[10];
  return B200_OK;
}

// check_convergence (termination_conditions.jl:339-372) for the plain modes and the Safe-mode state machine (:243-336);
// `du_norm` = ||u - uprev||_2
int term_check(b200_newton* nw, const TermQuant& q, double du_norm, bool* new_best) {
  TermCache& tc = nw->tc;
  *new_best = false;
  switch (tc.mode) {
    case B200_TERM_ABS_NORM: if (q.f_norm <= tc.abstol) { tc.retcode = B200_RC_SUCCESS; return 1; } return 0;
    case B200_TERM_ABS: if (q.f_inf <= tc.abstol) { tc.retcode = B200_RC_SUCCESS; return 1; } return 0;          // all(|du| <= abstol)
    case B200_TERM_NORM: if (q.f_norm <= tc.abstol || q.f_norm <= tc.reltol * q.sum_norm) { tc.retcode = B200_RC_SUCCESS; return 1; } return 0;
    case B200_TERM_REL_NORM: if (q.f_norm <= tc.reltol * q.sum_norm) { tc.retcode = B200_RC_SUCCESS; return 1; } return 0;
    case B200_TERM_REL: if (q.rel_viol == 0.0) { tc.retcode = B200_RC_SUCCESS; return 1; } return 0;          // all(|du| <= reltol |u + du|)
    default: break;
  }
  const bool rel = term_is_rel(tc.mode);
  double objective, criteria;
  if (!rel) { objective = q.f_norm; criteria = tc.abstol; }
  else { objective = q.f_norm / (q.sum_norm + (nextafter(tc.reltol, INFINITY) - tc.reltol)); criteria = tc.reltol; }  // + eps(reltol)
  if (!std::isfinite(objective)) { tc.retcode = B200_RC_UNSTABLE; return 1; }
  if (term_is_best(tc.mode) && objective < tc.best) { tc.best = objective; *new_best = true; }
  if (objective <= criteria) { tc.retcode = B200_RC_SUCCESS; return 1; }
  tc.nsteps += 1;
  tc.obj_trace[(tc.nsteps - 1) % 100] = objective;
  if (objective <= 3.0 * criteria && tc.nsteps > 100) {  // patience_objective_multiplier = 3, patience_steps = 100, min_max_factor = 1.3
    double mn = INFINITY, mx = -INFINITY;
    for (int i = 0; i < 100; ++i) { mn = std::min(mn, tc.obj_trace[i]); mx = std::max(mx, tc.obj_trace[i]); }
    if (mn < 1.3 * mx) { tc.retcode = B200_RC_STALLED; return 1; }
  }
  if (tc.max_stalled > 0) {
    tc.step_trace[(tc.nsteps - 1) % tc.max_stalled] = du_norm;
    if (tc.nsteps > tc.max_stalled) {
      double mx = 0.0;
      for (int i = 0; i < tc.max_stalled; ++i) mx = std::max(mx, tc.step_trace[i]);
      const bool stalled = rel ? (mx <= tc.reltol * (mx + tc.u0_norm)) : (mx <= tc.abstol);
      if (stalled) { tc.retcode = B200_RC_STALLED; return 1; }
    }
  }
  tc.retcode = B200_RC_FAILURE;
  return 0;
}

// A device buffer of `count` elements that b200_newton_destroy frees; B200_ERR_NOMEM saying `what` when it does not fit.
template <class T>
int32_t dev_alloc(b200_newton* nw, T** p, size_t count, const char* what) {
  if (cudaMalloc(p, sizeof(T) * count) != cudaSuccess) {
    cudaGetLastError();
    *p = nullptr;
    return nw->ctx->fail(B200_ERR_NOMEM, what, __FILE__, __LINE__);
  }
  nw->allocs.push_back(*p);
  return B200_OK;
}
// n-vectors, padded to an even length
int32_t dev_vecs(b200_newton* nw, std::initializer_list<double**> ps) {
  for (double** p : ps) B200_TRY(dev_alloc(nw, p, (size_t)((nw->n + 1) & ~(int64_t)1), "newton_create: the driver's n-vectors do not fit in device memory"));
  return B200_OK;
}

}  // namespace

extern "C" {
void b200_newton_opts_default(b200_newton_opts* o) {
  memset(o, 0, sizeof(*o));
  o->abstol = 0.0;  // => 3e-13
  o->reltol = 0.0;
  o->maxiters = 1000;
  o->linsolve = B200_LINSOLVE_GMRES;
  o->jvp_mode = B200_JVP_EXACT;
  o->globalization = B200_GLOBALIZATION_NONE;
  o->forcing = B200_FORCING_NONE;
  o->termination = B200_TERM_ABS_NORM_SAFE_BEST;
  o->store_trace = 1;
  o->fused_step = 1;
  b200_gmres_opts_default(&o->gmres);
  o->gmres.atol = 0.0;  // inherit the nonlinear tolerances (solve.jl:203)
  o->gmres.rtol = 0.0;
  o->ew_eta0 = 0.5; o->ew_eta_max = 0.9; o->ew_gamma = 0.9; o->ew_alpha = 2.0; o->ew_safeguard_threshold = 0.1; o->ew_safeguard = 1;
  o->max_shrink_times = 32;
}

int32_t b200_newton_destroy(b200_newton* nw) {
  B200_DEVICE_GUARD(nw ? nw->ctx : nullptr);
  if (!nw) return B200_OK;
  cudaStreamSynchronize(nw->ctx->stream);
  for (void* p : nw->allocs) cudaFree(p);
  if (nw->gm) b200_gmres_destroy(nw->gm);
  if (nw->mg) b200i_mg_destroy(nw->mg);
  if (nw->sj) b200_sparse_jac_destroy(nw->sj);
  if (nw->slu) b200_sparse_lu_destroy(nw->slu);
  if (nw->ilu) b200_ilu0_destroy(nw->ilu);
  if (nw->amg) b200_amg_destroy(nw->amg);
  delete nw;
  return B200_OK;
}

static bool ilu0_precond(const b200_newton_opts& o) { return o.precond == B200_PRECOND_ILU0_LEFT || o.precond == B200_PRECOND_ILU0_RIGHT; }
static bool sa_precond(const b200_newton_opts& o) { return o.precond == B200_PRECOND_SA_AMG_LEFT || o.precond == B200_PRECOND_SA_AMG_RIGHT; }
static bool amg_precond(const b200_newton_opts& o) { return o.precond == B200_PRECOND_AMG_LEFT || o.precond == B200_PRECOND_AMG_RIGHT || sa_precond(o); }

// the buffers and sub-solvers b200_newton_create builds for the options; on failure the caller destroys the partial driver
static int32_t newton_setup(b200_newton* nw) {
  b200_ctx* ctx = nw->ctx;
  b200_problem* prob = nw->prob;
  const b200_newton_opts& o = nw->o;
  const int64_t n = nw->n;
  B200_TRY(dev_vecs(nw, {&nw->u, &nw->fu, &nw->du, &nw->xlin}));
  if (term_is_best(o.termination)) B200_TRY(dev_vecs(nw, {&nw->best_u}));
  if (o.globalization == B200_GLOBALIZATION_TRUST_REGION)
    B200_TRY(dev_vecs(nw, {&nw->u_trial, &nw->fu_trial, &nw->Jdu, &nw->JTfu, &nw->du_c, &nw->c1, &nw->c2}));
  if (o.globalization == B200_GLOBALIZATION_LINESEARCH) B200_TRY(dev_vecs(nw, {&nw->u_trial, &nw->fu_trial, &nw->Jdu}));
  if (o.descent == B200_DESCENT_LEVENBERG_MARQUARDT) {
    B200_TRY(dev_vecs(nw, {&nw->u_trial, &nw->fu_trial, &nw->Jdu, &nw->lm_dtd, &nw->lm_v, &nw->lm_a, &nw->lm_vold, &nw->lm_rhs}));
    B200_TRY(dev_alloc(nw, &nw->lmA, (size_t)(n * n), "LevenbergMarquardt: J'J does not fit in device memory"));
  }
  if (o.descent == B200_DESCENT_BROYDEN) {
    B200_TRY(dev_vecs(nw, {&nw->qn_dfu, &nw->qn_dfu_reset}));
    if (o.qn_update_rule == B200_QN_UPDATE_KLEMENT) {
      B200_TRY(dev_vecs(nw, {&nw->kl_J}));  // diagonal structure: nothing n x n
    } else {
      B200_TRY(dev_vecs(nw, {&nw->qn_Jdfu, &nw->qn_w, &nw->qn_c}));
      if (o.qn_init_jacobian == B200_QN_INIT_LOW_RANK) {
        nw->lr_m = std::max(1, std::min(o.qn_threshold > 0 ? o.qn_threshold : 10, nw->maxiters));  // threshold = min(threshold, maxiters)
        const char* what = "LimitedMemoryBroyden: the low-rank factors do not fit in device memory";
        B200_TRY(dev_alloc(nw, &nw->lr_U, (size_t)(n * nw->lr_m), what));
        B200_TRY(dev_alloc(nw, &nw->lr_V, (size_t)(n * nw->lr_m), what));
        B200_TRY(dev_alloc(nw, &nw->lr_c, (size_t)nw->lr_m, what));
      } else {
        B200_TRY(dev_alloc(nw, &nw->qn_Jinv, (size_t)(n * n), "Broyden: the stored inverse Jacobian (n x n) does not fit in device memory"));
      }
    }
  }
  nw->op.ctx = ctx; nw->op.n = n;
  if (o.precond == B200_PRECOND_MULTIGRID_LEFT || o.precond == B200_PRECOND_MULTIGRID_RIGHT) B200_TRY(b200i_mg_create(prob, &nw->mg));
  if (o.linsolve == B200_LINSOLVE_GMRES || o.linsolve == B200_LINSOLVE_SPARSE_GMRES) {
    b200_gmres_opts g = o.gmres;
    if (g.atol <= 0) g.atol = nw->abstol;  // linsolve_kwargs = (; abstol, reltol)   solve.jl:203
    if (g.rtol <= 0) g.rtol = nw->reltol;
    nw->o.gmres = g;
    B200_TRY(b200_gmres_create(ctx, n, &g, &nw->gm));
  }
  if (o.linsolve == B200_LINSOLVE_GMRES) {
    nw->op.kind = LINOP_PROBLEM; nw->op.prob = prob; nw->op.u = nw->u; nw->op.jvp_mode = o.jvp_mode;
  } else if (o.linsolve == B200_LINSOLVE_DENSE_LU) {
    B200_TRY(dev_alloc(nw, &nw->Jdense, (size_t)(n * n), "dense Jacobian does not fit in device memory"));
    B200_TRY(dev_alloc(nw, &nw->ipiv, (size_t)n, "dense Jacobian does not fit in device memory"));
  } else if (o.linsolve == B200_LINSOLVE_SPARSE_GMRES || o.linsolve == B200_LINSOLVE_SPARSE_LU) {
    // jac_prototype + colouring once at init (jacobian.jl:286-353; colouring ext :13-28)
    int64_t nnz = 0;
    B200_TRY(b200_pattern_nnz(prob, &nnz));
    std::vector<int64_t> colptr(n + 1), rowval(nnz), colors(n);
    int64_t ncolors = 0;
    B200_TRY(b200_pattern(prob, 1, colptr.data(), rowval.data()));
    B200_TRY(b200_coloring_column(n, colptr.data(), rowval.data(), 1, B200_ORDER_LARGEST_FIRST, colors.data(), &ncolors));
    B200_TRY(b200_sparse_jac_create(prob, colptr.data(), rowval.data(), 1, colors.data(), ncolors, &nw->sj));
    B200_TRY(dev_alloc(nw, &nw->nzval, (size_t)nnz, "sparse Jacobian: the nonzero values do not fit in device memory"));
    // sparse direct route (linsolve = nothing on a sparse prototype): symbolic phase once, like LinearSolve's cache
    if (o.linsolve == B200_LINSOLVE_SPARSE_LU) B200_TRY(b200_sparse_lu_create(ctx, n, colptr.data(), rowval.data(), 1, &nw->slu));
    if (ilu0_precond(o)) B200_TRY(b200_ilu0_create(ctx, n, colptr.data(), rowval.data(), 1, &nw->ilu));
    if (sa_precond(o)) B200_TRY(b200_amg_create_sa(ctx, n, colptr.data(), rowval.data(), 1, nullptr, &nw->amg));
    else if (amg_precond(o)) B200_TRY(b200_amg_create(ctx, n, colptr.data(), rowval.data(), 1, nullptr, &nw->amg));
    nw->op.kind = LINOP_SPARSE_JAC; nw->op.sj = nw->sj; nw->op.nzval = nw->nzval;
  } else {
    return ctx->fail(B200_ERR_INVALID, "unknown linsolve kind", __FILE__, __LINE__);
  }
  return B200_OK;
}

int32_t b200_newton_create(b200_problem* prob, const b200_newton_opts* opts, b200_newton** out) {
  B200_DEVICE_GUARD(prob ? prob->ctx : nullptr);
  b200_ctx* ctx = prob->ctx;
  B200_REQUIRE(ctx, opts && out, "newton_create: bad arguments");
  B200_REQUIRE(ctx, opts->tr_scheme >= B200_TR_SIMPLE && opts->tr_scheme <= B200_TR_BASTIN, "newton_create: unknown radius update scheme");
  B200_REQUIRE(ctx, opts->termination >= B200_TERM_ABS_NORM_SAFE_BEST && opts->termination <= B200_TERM_REL_NORM_SAFE_BEST, "newton_create: unknown termination mode");
  B200_REQUIRE(ctx, opts->term_norm == B200_NORM_INF || opts->term_norm == B200_NORM_L2, "newton_create: unknown termination norm");
  B200_REQUIRE(ctx, opts->term_max_stalled_steps <= 128, "newton_create: term_max_stalled_steps must be <= 128");
  B200_REQUIRE(ctx, opts->descent == B200_DESCENT_NEWTON || (opts->descent == B200_DESCENT_PSEUDO_TRANSIENT && opts->globalization != B200_GLOBALIZATION_TRUST_REGION) ||
                        (opts->descent == B200_DESCENT_LEVENBERG_MARQUARDT && opts->globalization == B200_GLOBALIZATION_NONE && opts->linsolve == B200_LINSOLVE_DENSE_LU) ||
                        (opts->descent == B200_DESCENT_BROYDEN && opts->globalization == B200_GLOBALIZATION_NONE &&
                         (prob->n <= 65535 || opts->qn_init_jacobian == B200_QN_INIT_LOW_RANK || opts->qn_update_rule == B200_QN_UPDATE_KLEMENT) &&
                         (opts->qn_init_jacobian == B200_QN_INIT_IDENTITY || opts->qn_init_jacobian == B200_QN_INIT_LOW_RANK ||
                          (opts->qn_init_jacobian == B200_QN_INIT_TRUE_JACOBIAN && opts->linsolve == B200_LINSOLVE_DENSE_LU)) &&
                         (opts->qn_update_rule == B200_QN_UPDATE_GOOD_BROYDEN || opts->qn_update_rule == B200_QN_UPDATE_BAD_BROYDEN ||
                          (opts->qn_update_rule == B200_QN_UPDATE_KLEMENT && opts->qn_init_jacobian == B200_QN_INIT_IDENTITY))),
               "newton_create: descent must be Newton, PseudoTransient (without a trust region), LevenbergMarquardt (dense concrete Jacobian, its own trust region) or "
               "Broyden (no globalisation, n <= 65535, init_jacobian = true_jacobian needs the dense LU)");
  B200_REQUIRE(ctx, opts->precond >= B200_PRECOND_NONE && opts->precond <= B200_PRECOND_SA_AMG_RIGHT, "newton_create: unknown preconditioner");
  if (amg_precond(*opts)) {
    // AMG coarsens the assembled sparse Jacobian (any pattern); PseudoTransient's shift changes every step, as for ILU0
    B200_REQUIRE(ctx, opts->linsolve == B200_LINSOLVE_SPARSE_GMRES,
                 "newton_create: the AMG preconditioner coarsens the assembled sparse Jacobian: use concrete_jac = true (linsolve B200_LINSOLVE_SPARSE_GMRES)");
    if (opts->descent == B200_DESCENT_PSEUDO_TRANSIENT)
      return ctx->fail(B200_ERR_UNSUPPORTED, "newton_create: PseudoTransient with the AMG preconditioner is not offered (use block-Jacobi, multigrid or no preconditioner)", __FILE__, __LINE__);
  } else if (ilu0_precond(*opts)) {
    // ILU(0) factors the assembled sparse Jacobian, so any problem with a pattern qualifies; the SER shift of PseudoTransient
    // changes every step and would need a refactorisation every step, as on the sparse direct route
    B200_REQUIRE(ctx, opts->linsolve == B200_LINSOLVE_SPARSE_GMRES,
                 "newton_create: the ILU0 preconditioner factors the assembled sparse Jacobian: use concrete_jac = true (linsolve B200_LINSOLVE_SPARSE_GMRES)");
    if (opts->descent == B200_DESCENT_PSEUDO_TRANSIENT)
      return ctx->fail(B200_ERR_UNSUPPORTED, "newton_create: PseudoTransient with the ILU0 preconditioner is not offered (use block-Jacobi, multigrid or no preconditioner)", __FILE__, __LINE__);
  } else {
    B200_REQUIRE(ctx, opts->precond == B200_PRECOND_NONE ||
                          ((opts->linsolve == B200_LINSOLVE_GMRES || opts->linsolve == B200_LINSOLVE_SPARSE_GMRES) &&
                           (prob->kind == B200_PROB_BRUSS2D || prob->kind == B200_PROB_BRUSS3D)),
                 "newton_create: the built-in preconditioners need a Krylov linsolve and a built-in Brusselator problem");
  }
  b200_newton* nw = new b200_newton();
  nw->ctx = ctx; nw->prob = prob; nw->o = *opts; nw->n = prob->n;
  nw->abstol = opts->abstol > 0 ? opts->abstol : 3.0e-13;  // common_defaults.jl:44-48
  nw->reltol = opts->reltol > 0 ? opts->reltol : 3.0e-13;
  nw->maxiters = opts->maxiters > 0 ? opts->maxiters : 1000;
  nw->trp = b200i_tr_params(*opts);
  const int32_t s = newton_setup(nw);
  if (s != B200_OK) { b200_newton_destroy(nw); return s; }
  *out = nw;
  return B200_OK;
}

// reinit!(cache, u0): everything __init computes from u0 (solve.jl:191-284; termination_conditions.jl:134-179)
int32_t b200_newton_reinit(b200_newton* nw, const double* u0_dev) {
  B200_DEVICE_GUARD(nw ? nw->ctx : nullptr);
  b200_ctx* ctx = nw->ctx;
  const int64_t n = nw->n;
  const b200_newton_opts& o = nw->o;
  if (u0_dev != nw->u) CUDA_TRY(ctx, cudaMemcpyAsync(nw->u, u0_dev, sizeof(double) * n, cudaMemcpyDeviceToDevice, ctx->stream));
  nw->amg_built = 0;  // the first fresh Jacobian of this solve rebuilds the AMG hierarchy
  CUDA_TRY(ctx, cudaMemsetAsync(ctx->d_scalars, 0, sizeof(double) * 4, ctx->stream));
  B200_TRY(b200i_residual_norm(nw->prob, nw->u, nw->fu, ctx->d_scalars));  // evaluate_f(prob,u): nf is NOT bumped (solve.jl:194)
  CUDA_TRY(ctx, cudaMemsetAsync(nw->du, 0, sizeof(double) * n, ctx->stream));  // descent caches start with a defined du
  if (nw->best_u) CUDA_TRY(ctx, cudaMemcpyAsync(nw->best_u, nw->u, sizeof(double) * n, cudaMemcpyDeviceToDevice, ctx->stream));
  B200_TRY(b200i_fetch_scalars(ctx, 1));
  nw->fnorm_inf = ctx->h_scalars[0];
  memset(&nw->tc, 0, sizeof(nw->tc));
  nw->tc.mode = o.termination;
  nw->tc.norm_kind = o.term_norm;
  nw->tc.max_stalled = !term_is_safe(o.termination) ? 0 : (o.term_max_stalled_steps < 0 ? 0 : (o.term_max_stalled_steps == 0 ? 32 : o.term_max_stalled_steps));
  nw->tc.abstol = nw->abstol;
  nw->tc.reltol = nw->reltol;
  nw->total_time = 0.0;
  {  // SciMLBase.reinit!(::NonlinearTerminationModeCache, du, u)   termination_conditions.jl:180-215
    TermQuant q;
    B200_TRY(term_quantities(nw, nw->fu, nw->u, nw->fnorm_inf, &q));
    if (!term_is_safe(o.termination)) nw->tc.best = INFINITY;
    else if (!term_is_rel(o.termination)) nw->tc.best = q.f_norm;
    else {
      nw->tc.best = q.f_norm / (q.sum_norm + 2.220446049250313e-16);   // eps(TT)
      if (nw->tc.max_stalled > 0) B200_TRY(h_nrm2(nw, nw->u, &nw->tc.u0_norm));
    }
    nw->tc.initial = nw->tc.best;
  }
  memset(&nw->res, 0, sizeof(nw->res));
  nw->trace.clear();
  nw->retcode = B200_RC_DEFAULT; nw->force_stop = 0; nw->make_new_jacobian = 1; nw->nsteps = 0; nw->have_factor = 0;
  nw->shrink_counter = 0; nw->bytes = 2.0 * 8.0 * n;
  if (o.linsolve == B200_LINSOLVE_DENSE_LU) nw->res.njacs += 1;  // jac_prototype === nothing: DI.jacobian at init (jacobian.jl:103-117)
  if (o.globalization == B200_GLOBALIZATION_TRUST_REGION) {  // trust_region.jl:204-258, 330-346 (Simple scheme)
    double fu_norm, u0_norm, umin, umax;
    const int sch = o.tr_scheme;
    B200_TRY(h_nrm2(nw, nw->fu, &fu_norm));
    B200_TRY(h_nrm2(nw, nw->u, &u0_norm));
    B200_TRY(b200_extrema(ctx, n, nw->u, &umin, &umax));
    nw->tp1 = nw->trp.tp1; nw->tp2 = nw->trp.tp2; nw->tp3 = nw->trp.tp3; nw->tp4 = nw->trp.tp4;
    if (o.tr_max_trust_radius > 0) nw->max_tr = o.tr_max_trust_radius;  // max_trust_radius  :330-337
    else nw->max_tr = (sch == B200_TR_SIMPLE || sch == B200_TR_NOCEDAL_WRIGHT) ? std::max(fu_norm, umax - umin) : INFINITY;  // Hei, Yuan, Fan, NLsolve, Bastin: unbounded
    if (o.tr_initial_trust_radius > 0) nw->trust_region = o.tr_initial_trust_radius;  // initial_trust_radius  :339-346
    else if (sch == B200_TR_NLSOLVE) nw->trust_region = u0_norm > 0 ? u0_norm : 1.0;
    else if (sch == B200_TR_HEI || sch == B200_TR_BASTIN) nw->trust_region = 1.0;
    else if (sch == B200_TR_FAN) nw->trust_region = pow(fu_norm, 0.99) / 10.0;
    else nw->trust_region = nw->max_tr / 11.0;
    if (sch == B200_TR_YUAN) {  // itr = p1 ||J' fu||  :232-234
      double g;
      B200_TRY(b200_vjp(nw->prob, nw->u, nw->fu, nw->JTfu));
      B200_TRY(h_nrm2(nw, nw->JTfu, &g));
      nw->trust_region = nw->tp1 * g;
    }
  }
  if (o.descent == B200_DESCENT_PSEUDO_TRANSIENT) {  // SwitchedEvolutionRelaxationCache init / reinit! (pseudo_transient.jl:105-130)
    nw->alpha_inv = 1.0 / (o.pt_alpha_initial > 0 ? o.pt_alpha_initial : 1.0e-3);
    B200_TRY(h_nrm2(nw, nw->fu, &nw->pt_res_norm));
  }
  if (o.descent == B200_DESCENT_LEVENBERG_MARQUARDT) {  // LevenbergMarquardtDampingCache / TrustRegionCache init + reinit!  levenberg_marquardt.jl:71-117, 226-262
    nw->lm_lambda = o.lm_damping_initial > 0 ? o.lm_damping_initial : 1.0;
    nw->lm_lambda_factor = o.lm_damping_increase > 0 ? o.lm_damping_increase : 2.0;
    B200_TRY(b200_fill(ctx, n, o.lm_min_damping_D > 0 ? o.lm_min_damping_D : 1.0e-8, nw->lm_dtd));
    B200_TRY(b200_copy(ctx, n, nw->u, nw->lm_vold));   // `@bb v = copy(u)`: the previous velocity starts as u0
    B200_TRY(b200_fill(ctx, n, 0.0, nw->du));
    nw->lm_norm_v_old = INFINITY;
    nw->lm_loss_old = INFINITY;
  }
  if (o.descent == B200_DESCENT_BROYDEN) {  // BroydenUpdateRuleCache.dfu = copy(fu); NoChangeInStateResetCache.dfu = copy(fu); counters 0
    B200_TRY(b200_copy(ctx, n, nw->fu, nw->qn_dfu));
    B200_TRY(b200_copy(ctx, n, nw->fu, nw->qn_dfu_reset));
    B200_TRY(b200_fill(ctx, n, 0.0, nw->du));
    nw->qn_since_du = nw->qn_since_dfu = nw->qn_nresets = 0;
  }
  nw->op.shift = 0.0;
  nw->eta = o.ew_eta0;
  if (o.forcing == B200_FORCING_EW2) {
    B200_TRY(h_nrm2(nw, nw->fu, &nw->rnorm));
    nw->rnorm_prev = nw->rnorm;
  }
  nw->initialised = 1;
  return B200_OK;
}

// u += a du ; fu = f(u), with ||du||_2^2 and ||fu||_inf from the two kernels' epilogues, fetched together (solve.jl:403-407, 436-445)
static int32_t update_u(b200_newton* nw, double a, double* objective, double* du_norm) {
  b200_ctx* ctx = nw->ctx;
  CUDA_TRY(ctx, cudaMemsetAsync(ctx->d_scalars, 0, sizeof(double) * 2, ctx->stream));
  B200_TRY(b200i_axpy_norm(ctx, nw->n, a, nw->du, nw->u, ctx->d_scalars + 1));
  B200_TRY(b200i_residual_norm(nw->prob, nw->u, nw->fu, ctx->d_scalars));
  nw->res.nf += 1;
  B200_TRY(b200i_fetch_scalars(ctx, 2));
  *objective = ctx->h_scalars[0];
  *du_norm = sqrt(ctx->h_scalars[1]);
  return B200_OK;
}

// u_trial = u + a d
static int32_t trial_point(b200_newton* nw, double a, const double* d) {
  B200_TRY(b200_copy(nw->ctx, nw->n, nw->u, nw->u_trial));
  return b200_axpy(nw->ctx, nw->n, a, d, nw->u_trial);
}

// the trial point becomes the iterate: copyto!(cache.u, u_new) as a pointer swap
static void accept_trial(b200_newton* nw) {
  std::swap(nw->u, nw->u_trial);
  std::swap(nw->fu, nw->fu_trial);
  nw->op.u = nw->u;
}

// The end of every step: check_and_update! (the termination test on the iterate with ||f||_inf = objective, the best
// iterate), then update_trace!.  `t` carries the step's own fields (accepted, lin_*, trust_radius); LevenbergMarquardt
// skips the test (check = false) when its descent rejected the step.
static int32_t step_end(b200_newton* nw, double objective, double du_norm, b200_trace_rec t, bool check = true) {
  if (check) {
    nw->fnorm_inf = objective;
    bool new_best = false;
    TermQuant tq;
    B200_TRY(term_quantities(nw, nw->fu, nw->u, objective, &tq));
    if (term_check(nw, tq, du_norm, &new_best)) { nw->retcode = nw->tc.retcode; nw->force_stop = 1; }
    if (new_best && nw->best_u) CUDA_TRY(nw->ctx, cudaMemcpyAsync(nw->best_u, nw->u, sizeof(double) * nw->n, cudaMemcpyDeviceToDevice, nw->ctx->stream));
  }
  if (nw->o.store_trace) {
    t.iter = nw->nsteps + 1; t.fnorm_inf = objective; t.step_norm2 = du_norm;
    nw->trace.push_back(t);
  }
  return B200_OK;
}

// One step of LevenbergMarquardt() (levenberg_marquardt.jl; descent/damped_newton.jl :normal_form; descent/geodesic_acceleration.jl:
// 95-135; step! solve.jl:325-465).  All n-vectors and both n x n matrices stay on the device; the host takes the scalar
// decisions from a handful of norms / dots.
static int32_t lm_step(b200_newton* nw) {
  b200_ctx* ctx = nw->ctx;
  const int64_t n = nw->n;
  const b200_newton_opts& o = nw->o;
  const double inc = o.lm_damping_increase > 0 ? o.lm_damping_increase : 2.0, dec = o.lm_damping_decrease > 0 ? o.lm_damping_decrease : 3.0;
  const double h = o.lm_finite_diff_step > 0 ? o.lm_finite_diff_step : 0.1, alpha_geo = o.lm_alpha_geodesic > 0 ? o.lm_alpha_geodesic : 0.75;
  const double b_uphill = o.lm_b_uphill > 0 ? o.lm_b_uphill : (o.lm_b_uphill == 0 ? 1.0 : 0.0);
  if (nw->make_new_jacobian) {  // J = cache.jac_cache(u)
    nw->res.njacs += 1;
    B200_TRY(b200_dense_jac_fill(nw->prob, nw->u, nw->Jdense, n));
  }
  // ---- DampedNewtonDescent, normal form: A = J'J + lambda D'D with D'D = running max of diag(J'J); v = -(A^-1 J' f)
  B200_TRY(b200i_gram(ctx, n, nw->Jdense, n, nw->lmA, n));
  B200_TRY(b200i_lm_damp(ctx, n, nw->lmA, n, nw->lm_dtd, nw->lm_lambda));
  int32_t info = 0;
  nw->res.nfactors += 1;
  B200_TRY(b200_getrf(ctx, n, nw->lmA, n, nw->ipiv, &info));
  int descent_ok = 1, tr_ok = 0, accepted = 0;
  double objective = nw->fnorm_inf, du_norm = 0.0;
  if (info != 0) {  // the damped normal matrix is singular: LinearSolve failure with a current Jacobian
    if (nw->make_new_jacobian) { nw->retcode = B200_RC_INTERNAL_LINSOLVE_FAILED; nw->force_stop = 1; return B200_OK; }
    nw->make_new_jacobian = 1;
    return lm_step(nw);
  }
  B200_TRY(b200_gemv(ctx, 1, n, n, nw->Jdense, n, nw->fu, nw->lm_rhs));          // J' f
  B200_TRY(b200_copy(ctx, n, nw->lm_rhs, nw->lm_v));
  nw->res.nsolve += 1;
  B200_TRY(b200_getrs(ctx, n, 1, nw->lmA, n, nw->ipiv, nw->lm_v, n));
  B200_TRY(b200_scal(ctx, n, -1.0, nw->lm_v));
  double norm_v;
  B200_TRY(h_nrm2(nw, nw->lm_v, &norm_v));
  if (!o.lm_disable_geodesic) {
    // geodesic acceleration: fu_cache = (2/h) ((f(u + h v) - f(u)) / h - J v) ; a = -(A^-1 J' fu_cache) with the same factorisation
    B200_TRY(trial_point(nw, h, nw->lm_v));
    B200_TRY(b200_residual(nw->prob, nw->u_trial, nw->fu_trial));              // evaluate_f!! inside the descent: NLStats.nf is not bumped
    B200_TRY(b200_gemv(ctx, 0, n, n, nw->Jdense, n, nw->lm_v, nw->Jdu));        // J v
    B200_TRY(b200_axpy(ctx, n, -1.0, nw->fu, nw->fu_trial));
    B200_TRY(b200_axpby(ctx, n, -2.0 / h, nw->Jdu, 2.0 / (h * h), nw->fu_trial));
    B200_TRY(b200_gemv(ctx, 1, n, n, nw->Jdense, n, nw->fu_trial, nw->lm_a));
    nw->res.nsolve += 1;
    B200_TRY(b200_getrs(ctx, n, 1, nw->lmA, n, nw->ipiv, nw->lm_a, n));
    B200_TRY(b200_scal(ctx, n, -1.0, nw->lm_a));
    double norm_a;
    B200_TRY(h_nrm2(nw, nw->lm_a, &norm_a));
    if (2.0 * norm_a <= norm_v * alpha_geo) {
      B200_TRY(b200_copy(ctx, n, nw->lm_v, nw->du));
      B200_TRY(b200_axpy(ctx, n, 0.5, nw->lm_a, nw->du));                       // du = v + a / 2
    } else {
      descent_ok = 0;  // the step is not taken; du keeps its previous value (geodesic_acceleration.jl:131-133)
    }
  } else {
    B200_TRY(b200_copy(ctx, n, nw->lm_v, nw->du));
  }
  nw->make_new_jacobian = 0;
  if (descent_ok) {
    // ---- LevenbergMarquardtTrustRegion: beta = cos(v, v_old); accept iff (1 - beta)^b_uphill * ||f(u + du)|| <= loss_old
    double vdot;
    B200_TRY(h_dot(nw, nw->lm_v, nw->lm_vold, &vdot));
    const double beta = vdot / (norm_v * nw->lm_norm_v_old);
    B200_TRY(trial_point(nw, 1.0, nw->du));
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->d_scalars, 0, sizeof(double) * 2, ctx->stream));
    B200_TRY(b200i_residual_norm(nw->prob, nw->u_trial, nw->fu_trial, ctx->d_scalars));
    nw->res.nf += 1;
    B200_TRY(b200i_fetch_scalars(ctx, 1));
    const double trial_inf = ctx->h_scalars[0];
    double loss;
    B200_TRY(h_nrm2(nw, nw->fu_trial, &loss));
    tr_ok = (pow(1.0 - beta, b_uphill) * loss <= nw->lm_loss_old) ? 1 : 0;     // loss_old is never updated by the reference (stays Inf)
    if (tr_ok) {
      nw->make_new_jacobian = 1;
      nw->lm_norm_v_old = norm_v;
      B200_TRY(b200_copy(ctx, n, nw->lm_v, nw->lm_vold));
      B200_TRY(h_nrm2(nw, nw->du, &du_norm));
      accept_trial(nw);
      objective = trial_inf;
      accepted = 1;
    }
  }
  b200_trace_rec t = {};
  t.accepted = accepted; t.lin_status = descent_ok; t.trust_radius = nw->lm_lambda;  // the damping USED by this step
  B200_TRY(step_end(nw, objective, du_norm, t, descent_ok));
  // callback_into_cache! (levenberg_marquardt.jl:176-185): lambda shrinks after a step both the descent and the trust region accepted
  if (descent_ok && tr_ok) nw->lm_lambda_factor = 1.0 / dec;
  nw->lm_lambda *= nw->lm_lambda_factor;
  nw->lm_lambda_factor = inc;
  return B200_OK;
}

// Utils.initial_jacobian_scaling_alpha(alpha, u, fu, L2) of Broyden, LimitedMemoryBroyden and Klement: the given alpha, else
// 2 ||f|| / max(||u||, 1); 1 below ||f|| = 1e-5
static int32_t qn_initial_alpha(b200_newton* nw, double* alpha) {
  *alpha = nw->o.qn_alpha;
  if (*alpha > 0) return B200_OK;
  double fn, un;
  B200_TRY(h_nrm2(nw, nw->fu, &fn));
  B200_TRY(h_nrm2(nw, nw->u, &un));
  *alpha = (fn < 1.0e-5) ? 1.0 : (2.0 * fn) / std::max(un, 1.0);
  return B200_OK;
}

// One step of Broyden() (NonlinearSolveQuasiNewton/src/solve.jl:293-486, broyden.jl:124-144, reset_conditions.jl:52-88,
// initialization.jl:78-105).  The stored inverse J^-1 (n x n, column-major) lives in HBM; a step is GEMV-shaped:
//   du = -(J^-1 f)                               1 pass over J^-1
//   J^-1 += ((du - J^-1 df) / denom) w'          good Broyden: w = J^-T du, denom = <du, J^-1 df>   -> 2 GEMV + 1 GER = 4 passes
//                                                bad Broyden : w = df,      denom = ||df||^2        -> 1 GEMV + 1 GER = 3 passes
// The host takes the scalar decisions (reset counters, max_resets, termination) from a handful of reductions.
static int32_t broyden_init_inverse(b200_newton* nw) {
  b200_ctx* ctx = nw->ctx;
  const int64_t n = nw->n;
  if (nw->o.qn_init_jacobian == B200_QN_INIT_TRUE_JACOBIAN) {  // J^-1 = J \ I through the LU (Utils.linsolve_identity!!)
    nw->res.njacs += 1;
    B200_TRY(b200_dense_jac_fill(nw->prob, nw->u, nw->Jdense, n));
    int32_t info = 0;
    nw->res.nfactors += 1;
    B200_TRY(b200_getrf(ctx, n, nw->Jdense, n, nw->ipiv, &info));
    if (info != 0) { nw->retcode = B200_RC_INTERNAL_LINSOLVE_FAILED; nw->force_stop = 1; return B200_OK; }
    B200_TRY(b200i_scaled_identity(ctx, n, nw->qn_Jinv, n, 1.0));
    B200_TRY(b200_getrs(ctx, n, n, nw->Jdense, n, nw->ipiv, nw->qn_Jinv, n));
    return B200_OK;
  }
  double alpha;
  B200_TRY(qn_initial_alpha(nw, &alpha));
  if (nw->o.qn_init_jacobian == B200_QN_INIT_LOW_RANK) {  // BroydenLowRankJacobian: idx = 0, alpha = inv(scaling)   initialization.jl:176-199
    nw->lr_idx = 0;
    nw->lr_alpha = 1.0 / alpha;
    return B200_OK;
  }
  return b200i_scaled_identity(ctx, n, nw->qn_Jinv, n, 1.0 / alpha);
}

// y = J^-1 x (transpose = 0) or J^-T x (1): the dense stored inverse, or alpha x + U (V' x) resp. alpha x + V (U' x) for the low-rank form
static int32_t broyden_apply(b200_newton* nw, int transpose, const double* x, double* y) {
  b200_ctx* ctx = nw->ctx;
  const int64_t n = nw->n;
  if (nw->o.qn_init_jacobian != B200_QN_INIT_LOW_RANK) return b200_gemv(ctx, transpose, n, n, nw->qn_Jinv, n, x, y);
  const int k = std::min(nw->lr_idx, nw->lr_m);
  if (k > 0) {
    const double *L = transpose ? nw->lr_V : nw->lr_U, *R = transpose ? nw->lr_U : nw->lr_V;
    B200_TRY(b200_gemv(ctx, 1, n, k, R, n, x, nw->lr_c));   // c = R' x   (k dot products)
    B200_TRY(b200_gemv(ctx, 0, n, k, L, n, nw->lr_c, y));   // y = L c
    return b200_axpy(ctx, n, nw->lr_alpha, x, y);
  }
  return b200_axpby(ctx, n, nw->lr_alpha, x, 0.0, y);
}

static int32_t broyden_count(b200_newton* nw, const double* x, const double* y, double tol, double* out) {
  b200_ctx* ctx = nw->ctx;
  B200_TRY(b200i_reduce_sum_dev(ctx, nw->n, x, y, y ? RED_COUNT_DIFF_LE : RED_COUNT_LE, ctx->d_scalars, tol));
  B200_TRY(b200i_fetch_scalars(ctx, 1));
  *out = ctx->h_scalars[0];
  return B200_OK;
}

// One step of Klement() with its default diagonal structure (klement.jl:30-49, 128-140; reset_conditions.jl:103-120; solve.jl:293-486):
// J is an n-vector, so descent, update and the reset test are elementwise kernels and one counting reduction — any n.
static int32_t klement_step(b200_newton* nw) {
  b200_ctx* ctx = nw->ctx;
  const int64_t n = nw->n;
  const int max_resets = nw->o.qn_max_resets > 0 ? nw->o.qn_max_resets : 100;
  auto init_diag = [&]() -> int32_t {
    double alpha;
    B200_TRY(qn_initial_alpha(nw, &alpha));
    return b200_fill(ctx, n, alpha, nw->kl_J);   // J = one.(fu) .* alpha, NOT inverted (store_inverse_jacobian = false)
  };
  int reset = 0;
  if (nw->nsteps == 0) {
    B200_TRY(init_diag());
  } else {
    double zeros;  // IllConditionedJacobianReset on a Diagonal: any(iszero, diag(J))
    B200_TRY(broyden_count(nw, nw->kl_J, nullptr, 0.0, &zeros));
    if (zeros > 0) {
      reset = 1;
      if (++nw->qn_nresets >= max_resets) { nw->retcode = B200_RC_CONVERGENCE_FAILURE; nw->force_stop = 1; return B200_OK; }
      B200_TRY(init_diag());
    }
  }
  B200_TRY(b200i_klement_descent(ctx, n, nw->kl_J, nw->fu, nw->du));
  double objective, du_norm;
  B200_TRY(update_u(nw, 1.0, &objective, &du_norm));
  nw->res.nsolve += 1;   // the diagonal system goes through NativeJLLinearSolveCache (linear_solve.jl:130-134): nsolve and nfactors both +1
  nw->res.nfactors += 1;
  nw->bytes += 8.0 * (double)n * 8.0;
  b200_trace_rec t = {};
  t.accepted = 1; t.lin_status = reset;
  B200_TRY(step_end(nw, objective, du_norm, t));
  if (nw->force_stop) return B200_OK;
  return b200i_klement_update(ctx, n, nw->kl_J, nw->fu, nw->qn_dfu, nw->du);
}

static int32_t broyden_step(b200_newton* nw) {
  if (nw->o.qn_update_rule == B200_QN_UPDATE_KLEMENT) return klement_step(nw);
  b200_ctx* ctx = nw->ctx;
  const int64_t n = nw->n;
  const b200_newton_opts& o = nw->o;
  const double tol = o.qn_reset_tolerance > 0 ? o.qn_reset_tolerance : 1.8189894035458565e-12;  // eps^(3/4)
  const int max_resets = o.qn_max_resets > 0 ? o.qn_max_resets : 100;
  int reset = 0;
  if (nw->nsteps == 0) {
    B200_TRY(broyden_init_inverse(nw));
    if (nw->force_stop) return B200_OK;
  } else {
    // NoChangeInStateReset(nsteps = 3): ANY component of du (then of f - f_prev) at or below the tolerance counts as "no change"
    double cnt;
    B200_TRY(broyden_count(nw, nw->du, nullptr, tol, &cnt));
    if (cnt > 0) {
      if (++nw->qn_since_du >= 3) { nw->qn_since_du = nw->qn_since_dfu = 0; reset = 1; }
    } else {
      nw->qn_since_du = nw->qn_since_dfu = 0;
    }
    if (!reset) {
      B200_TRY(broyden_count(nw, nw->fu, nw->qn_dfu_reset, tol, &cnt));
      if (cnt > 0) {
        if (++nw->qn_since_dfu >= 3) { nw->qn_since_dfu = nw->qn_since_du = 0; reset = 1; }
      } else {
        nw->qn_since_dfu = nw->qn_since_du = 0;
      }
      B200_TRY(b200_copy(ctx, n, nw->fu, nw->qn_dfu_reset));
    }
    if (reset) {
      if (++nw->qn_nresets >= max_resets) { nw->retcode = B200_RC_CONVERGENCE_FAILURE; nw->force_stop = 1; return B200_OK; }
      B200_TRY(broyden_init_inverse(nw));
      if (nw->force_stop) return B200_OK;
    }
  }
  // ---- NewtonDescent on the stored inverse: du = -(J^-1 f) ; u += du ; f = f(u)
  B200_TRY(broyden_apply(nw, 0, nw->fu, nw->du));
  B200_TRY(b200_scal(ctx, n, -1.0, nw->du));
  double objective, du_norm;
  B200_TRY(update_u(nw, 1.0, &objective, &du_norm));
  const double pass_bytes = (o.qn_init_jacobian == B200_QN_INIT_LOW_RANK) ? 16.0 * (double)n * std::min(nw->lr_idx, nw->lr_m) : 8.0 * (double)n * (double)n;  // one product with the stored inverse
  nw->bytes += pass_bytes;
  b200_trace_rec t = {};
  t.accepted = 1; t.lin_status = reset;  // lin_status: J^-1 was re-initialised before this step
  B200_TRY(step_end(nw, objective, du_norm, t));
  if (nw->force_stop) return B200_OK;  // the reference skips the update once the step has stopped the solve
  // ---- update rule
  double* dfu = nw->qn_dfu;
  B200_TRY(b200_axpby(ctx, n, 1.0, nw->fu, -1.0, dfu));                  // dfu = fu - dfu
  B200_TRY(broyden_apply(nw, 0, dfu, nw->qn_Jdfu));                      // J^-1 dfu
  double denom;
  const double* rmul;
  if (o.qn_update_rule == B200_QN_UPDATE_GOOD_BROYDEN) {
    B200_TRY(broyden_apply(nw, 1, nw->du, nw->qn_w));                    // J^-T du
    B200_TRY(h_dot(nw, nw->du, nw->qn_Jdfu, &denom));
    rmul = nw->qn_w;
  } else {
    double nd;
    B200_TRY(h_nrm2(nw, dfu, &nd));
    denom = nd * nd;
    rmul = dfu;
  }
  const double inv = 1.0 / (denom == 0.0 ? 1.0e-5 : denom);
  double* c = nw->qn_c;
  B200_TRY(b200_copy(ctx, n, nw->du, c));
  B200_TRY(b200_axpy(ctx, n, -1.0, nw->qn_Jdfu, c));
  B200_TRY(b200_scal(ctx, n, inv, c));                                   // (du - J^-1 dfu) / denom
  if (o.qn_init_jacobian == B200_QN_INIT_LOW_RANK) {                      // mul!(J, u, v', true, true): the pair goes into slot idx mod m
    const int slot = nw->lr_idx % nw->lr_m;
    B200_TRY(b200_copy(ctx, n, c, nw->lr_U + (int64_t)slot * n));
    B200_TRY(b200_copy(ctx, n, rmul, nw->lr_V + (int64_t)slot * n));
    nw->lr_idx += 1;
  } else {
    B200_TRY(b200i_ger(ctx, n, nw->qn_Jinv, n, c, rmul));                // J^-1 += c rmul'
  }
  B200_TRY(b200_copy(ctx, n, nw->fu, dfu));
  nw->bytes += pass_bytes * (o.qn_update_rule == B200_QN_UPDATE_GOOD_BROYDEN ? 4.0 : 3.0);
  return B200_OK;
}

static bool krylov_linsolve(const b200_newton_opts& o) { return o.linsolve == B200_LINSOLVE_GMRES || o.linsolve == B200_LINSOLVE_SPARSE_GMRES; }

// J = cache.jac_cache(u) when the step asks for one (solve.jl:338-344); *fresh: the step works with a new Jacobian
static int32_t refresh_jacobian(b200_newton* nw, bool* fresh) {
  *fresh = nw->make_new_jacobian != 0;
  if (!*fresh || nw->o.linsolve == B200_LINSOLVE_GMRES) return B200_OK;  // matrix-free: nothing to assemble
  nw->res.njacs += 1;
  nw->have_factor = 0;
  if (nw->o.linsolve == B200_LINSOLVE_DENSE_LU) return b200_dense_jac_fill(nw->prob, nw->u, nw->Jdense, nw->n);  // written straight into the LU workspace (K10: no copyto!)
  B200_TRY(b200_sparse_jac_fill(nw->sj, nw->u, nw->nzval));
  // precs(A, p) on the new A; not an NLStats factorisation (LinearSolve's Krylov route counts none)
  if (nw->ilu) B200_TRY(b200_ilu0_factor(nw->ilu, nw->nzval, &nw->ilu_info));
  if (nw->amg) {  // the splitting is chosen once per solve; later Jacobians refresh the values on the device
    B200_TRY(b200_amg_setup(nw->amg, nw->nzval, !nw->amg_built, &nw->amg_info));
    nw->amg_built = nw->amg_info == 0;
  }
  return B200_OK;
}

// What precedes each linear solve: the PseudoTransient shift (its SER update once per step, on the first attempt) and the
// Eisenstat-Walker forcing (every attempt)
static int32_t pre_step(b200_newton* nw, bool first_attempt, bool fresh) {
  const b200_newton_opts& o = nw->o;
  if (o.descent == B200_DESCENT_PSEUDO_TRANSIENT && first_attempt) {
    // SER (pseudo_transient.jl:157-170): alpha^-1 *= ||f_n|| / ||f_{n-1}||  (2-norm); A = J + alpha^-1 I
    double rn;
    B200_TRY(h_nrm2(nw, nw->fu, &rn));
    nw->alpha_inv *= rn / nw->pt_res_norm;
    nw->pt_res_norm = rn;
    nw->op.shift = nw->alpha_inv;
  }
  if (o.descent == B200_DESCENT_PSEUDO_TRANSIENT && o.linsolve == B200_LINSOLVE_DENSE_LU && fresh)
    B200_TRY(b200i_diag_shift(nw->ctx, nw->n, nw->Jdense, nw->n, nw->alpha_inv));  // dampen_jacobian!!: J[i,i] += alpha^-1
  if (o.forcing == B200_FORCING_EW2 && krylov_linsolve(o)) {  // pre_step_forcing!   eisenstat_walker.jl:42-80
    if (nw->nsteps == 0) {
      nw->eta = o.ew_eta0;
      B200_TRY(h_nrm2(nw, nw->fu, &nw->rnorm));
      nw->rnorm_prev = nw->rnorm;
    } else {
      const double eta_prev = nw->eta;
      nw->eta = o.ew_gamma * pow(nw->rnorm / nw->rnorm_prev, o.ew_alpha);
      if (o.ew_safeguard) {
        const double sg = o.ew_gamma * pow(eta_prev, o.ew_alpha);
        if (sg > o.ew_safeguard_threshold && sg > nw->eta) nw->eta = sg;
      }
      nw->eta = std::min(std::max(nw->eta, 0.0), o.ew_eta_max);
    }
    B200_TRY(b200_gmres_set_tolerances(nw->gm, -1.0, nw->eta));  // LinearSolve.update_tolerances!(lincache; reltol = eta)
  }
  return B200_OK;
}

// J xlin = fu (newton.jl:97-141) by the sparse band LU, the dense LU (with its QR rescue) or GMRES; *ok = false is a
// LinearSolve failure.  *gs holds the GMRES statistics (zero for the direct solvers).
static int32_t linear_solve(b200_newton* nw, bool fresh, bool* ok, b200_gmres_stats* gs) {
  b200_ctx* ctx = nw->ctx;
  const int64_t n = nw->n;
  const b200_newton_opts& o = nw->o;
  *ok = true;
  memset(gs, 0, sizeof(*gs));
  nw->res.nsolve += 1;
  if (o.linsolve == B200_LINSOLVE_SPARSE_LU) {
    if (!nw->have_factor) {
      nw->res.nfactors += 1;
      int32_t info = 0;
      if (o.descent == B200_DESCENT_PSEUDO_TRANSIENT) return ctx->fail(B200_ERR_UNSUPPORTED, "PseudoTransient with the sparse direct solver is not offered (use dense LU or GMRES)", __FILE__, __LINE__);
      B200_TRY(b200_sparse_lu_factor(nw->slu, nw->nzval, &info));
      nw->have_factor = 1;
      if (info != 0) *ok = false;
    }
    if (*ok) B200_TRY(b200_sparse_lu_solve(nw->slu, nw->fu, nw->xlin));
  } else if (!krylov_linsolve(o)) {
    if (!nw->have_factor) {  // update_A! for a factorisation on a fresh A (…LinearSolveExt.jl:81-86)
      nw->res.nfactors += 1;
      int32_t info = 0;
      B200_TRY(b200_getrf(ctx, n, nw->Jdense, n, nw->ipiv, &info));
      nw->have_factor = 1;
      if (info != 0) *ok = false;
    }
    CUDA_TRY(ctx, cudaMemcpyAsync(nw->xlin, nw->fu, sizeof(double) * n, cudaMemcpyDeviceToDevice, ctx->stream));
    if (*ok) B200_TRY(b200_getrs(ctx, n, 1, nw->Jdense, n, nw->ipiv, nw->xlin, n));
    else if (n <= 4096) {
      // singular LU: LinearSolve's default dense solver falls back to a column-pivoted QR (linear_solve.jl:48-55).  The
      // factorisation destroyed J: refill it, solve in the least-squares sense (basic solution of the numerical-rank system).
      B200_TRY(b200_dense_jac_fill(nw->prob, nw->u, nw->Jdense, n));
      if (o.descent == B200_DESCENT_PSEUDO_TRANSIENT) B200_TRY(b200i_diag_shift(ctx, n, nw->Jdense, n, nw->alpha_inv));
      if (!nw->qr_work) {
        B200_TRY(dev_alloc(nw, &nw->qr_work, (size_t)(3 * n + 2), "QR rescue of a singular LU: the workspace does not fit in device memory"));
        B200_TRY(dev_alloc(nw, &nw->qr_jpvt, (size_t)(n + 2), "QR rescue of a singular LU: the workspace does not fit in device memory"));
      }
      CUDA_TRY(ctx, cudaMemcpyAsync(nw->qr_work + 2 * n, nw->fu, sizeof(double) * n, cudaMemcpyDeviceToDevice, ctx->stream));
      int32_t rank = 0;
      B200_TRY(b200i_qrcp_solve(ctx, n, nw->Jdense, n, nw->qr_work + 2 * n, nw->xlin, nw->qr_work, nw->qr_jpvt, &rank));
      nw->have_factor = 0;  // Jdense now holds the QR factors: the next step refactorises whatever happens
      *ok = rank > 0;
    }
  } else {
    // `linu` aliases the du buffer: it is the initial guess only when warm_start is requested
    if (o.gmres.warm_start) CUDA_TRY(ctx, cudaMemcpyAsync(nw->xlin, nw->du, sizeof(double) * n, cudaMemcpyDeviceToDevice, ctx->stream));
    if (nw->ilu && nw->ilu_info != 0) { *ok = false; return B200_OK; }  // zero pivot: a failed solve, retried with a fresh Jacobian
    if (nw->amg && nw->amg_info != 0) { *ok = false; return B200_OK; }  // zero diagonal or pivot: likewise
    if (o.precond != B200_PRECOND_NONE) {  // precs(A, p): rebuilt from the current iterate, like update_A! does for Pl / Pr
      memset(&nw->prec, 0, sizeof(nw->prec));
      nw->prec.ctx = ctx; nw->prec.n = n; nw->prec.prob = nw->prob; nw->prec.u = nw->u;
      if (nw->mg) {
        nw->prec.kind = LINOP_MULTIGRID; nw->prec.mg = nw->mg;
        if (fresh) B200_TRY(b200i_mg_setup(nw->mg, nw->u));  // coarse operators follow the linearisation point
      } else if (nw->ilu) {
        nw->prec.kind = LINOP_ILU0; nw->prec.ilu = nw->ilu;  // factorised by refresh_jacobian
      } else if (nw->amg) {
        nw->prec.kind = LINOP_AMG; nw->prec.amg = nw->amg;   // set up by refresh_jacobian
      } else {
        nw->prec.kind = LINOP_BLOCK_JACOBI;
      }
      const bool left = o.precond == B200_PRECOND_BLOCK_JACOBI_LEFT || o.precond == B200_PRECOND_MULTIGRID_LEFT || o.precond == B200_PRECOND_ILU0_LEFT ||
                        o.precond == B200_PRECOND_AMG_LEFT || o.precond == B200_PRECOND_SA_AMG_LEFT;
      B200_TRY(b200_gmres_set_precond(nw->gm, left ? &nw->prec : nullptr, left ? nullptr : &nw->prec));
    }
    B200_TRY(b200_gmres_solve(nw->gm, &nw->op, nw->fu, nw->xlin, gs));
    nw->res.njvp += gs->nmatvec;
    nw->bytes += gs->bytes;
    if (gs->status == B200_LS_NONFINITE || gs->status == B200_LS_OUT_OF_MEMORY) *ok = false;  // LinearSolve retcode Failure
  }
  return B200_OK;
}

// Dogleg (dogleg.jl:86-151): du holds the Newton step on entry and the dogleg step on return.  When the step is the Cauchy
// direction cut at the radius, ||J du||^2 is already known: *have_dJJd is set and *dJJd holds it.
static int32_t dogleg(b200_newton* nw, bool* have_dJJd, double* dJJd) {
  b200_ctx* ctx = nw->ctx;
  const int64_t n = nw->n;
  *have_dJJd = false;
  double nrm_newton;
  B200_TRY(h_nrm2(nw, nw->du, &nrm_newton));
  if (nrm_newton <= nw->trust_region) return B200_OK;
  B200_TRY(b200_vjp(nw->prob, nw->u, nw->fu, nw->du_c));  // du_c = -J' fu  (steepest.jl:60-80)
  B200_TRY(b200_scal(ctx, n, -1.0, nw->du_c));
  double l_grad, quad;
  B200_TRY(h_nrm2(nw, nw->du_c, &l_grad));
  B200_TRY(b200_jvp(nw->prob, nw->u, nw->du_c, nw->Jdu));
  B200_TRY(h_dot(nw, nw->Jdu, nw->Jdu, &quad));
  const double d_cauchy = (l_grad * l_grad * l_grad) / quad;
  if (d_cauchy >= nw->trust_region) {
    const double lam = nw->trust_region / l_grad;
    B200_TRY(b200_axpby(ctx, n, lam, nw->du_c, 0.0, nw->du));
    *have_dJJd = true;
    *dJJd = lam * lam * quad;
    return B200_OK;
  }
  B200_TRY(b200_axpby(ctx, n, d_cauchy / l_grad, nw->du_c, 0.0, nw->c1));  // c1 = (d_cauchy/l_grad) du_c
  B200_TRY(b200_copy(ctx, n, nw->du, nw->c2));
  B200_TRY(b200_axpy(ctx, n, -1.0, nw->c1, nw->c2));                         // c2 = du_newton - c1
  B200_TRY(b200i_reduce_sum_dev(ctx, n, nw->c2, nw->c2, RED_DOT, ctx->d_scalars));
  B200_TRY(b200i_reduce_sum_dev(ctx, n, nw->c1, nw->c2, RED_DOT, ctx->d_scalars + 1));
  B200_TRY(b200i_fetch_scalars(ctx, 2));
  const double a = ctx->h_scalars[0], b2 = ctx->h_scalars[1];
  const double b = 2.0 * b2, c = d_cauchy * d_cauchy - nw->trust_region * nw->trust_region;
  const double aux = std::max(0.0, b * b - 4.0 * a * c);
  const double tau = (-b + sqrt(aux)) / (2.0 * a);
  B200_TRY(b200_copy(ctx, n, nw->c1, nw->du));
  return b200_axpy(ctx, n, tau, nw->c2, nw->du);
}

// solve.jl:392-408 with LineSearch.jl BackTracking (cubic interpolation; external package restated, see oracle.c):
// phi(a) = ||f(u + a du)||^2 / 2, phi'(0) = <fu, J du> by one JVP; every trial is one axpby + one residual + one norm.
// *alpha is the step length to take; a search that runs out of iterations stops the solve with LINESEARCH_FAILED.
static int32_t backtracking(b200_newton* nw, double* alpha) {
  const b200_newton_opts& o = nw->o;
  const double c1 = o.ls_c1 > 0 ? o.ls_c1 : 1e-4, rho_hi = o.ls_rho_hi > 0 ? o.ls_rho_hi : 0.5, rho_lo = o.ls_rho_lo > 0 ? o.ls_rho_lo : 0.1;
  const int ls_max = o.ls_maxiters > 0 ? o.ls_maxiters : 1000;
  double nf0, dphi0;
  B200_TRY(h_nrm2(nw, nw->fu, &nf0));
  const double phi0 = 0.5 * nf0 * nf0;
  B200_TRY(b200_jvp(nw->prob, nw->u, nw->du, nw->Jdu));
  B200_TRY(h_dot(nw, nw->fu, nw->Jdu, &dphi0));
  auto phi = [&](double a, double* out) -> int32_t {
    B200_TRY(trial_point(nw, a, nw->du));
    B200_TRY(b200_residual(nw->prob, nw->u_trial, nw->fu_trial));
    nw->res.nf += 1;
    double t;
    B200_TRY(h_nrm2(nw, nw->fu_trial, &t));
    *out = 0.5 * t * t;
    return B200_OK;
  };
  double a1 = 1.0, a2 = 1.0, phx0 = phi0, phx1;
  B200_TRY(phi(a1, &phx1));
  int itf = 0;
  while (!std::isfinite(phx1) && itf < 50) { ++itf; a1 = a2; a2 = a1 / 2.0; B200_TRY(phi(a2, &phx1)); }
  int it = 0;
  while (phx1 > phi0 + c1 * a2 * dphi0) {
    if (++it > ls_max) { nw->retcode = B200_RC_INTERNAL_LINESEARCH_FAILED; nw->force_stop = 1; break; }
    double at;
    if (it == 1) at = -(dphi0 * a2 * a2) / (2.0 * (phx1 - phi0 - dphi0 * a2));
    else {
      const double div = 1.0 / (a1 * a1 * a2 * a2 * (a2 - a1));
      const double ca = (a1 * a1 * (phx1 - phi0 - dphi0 * a2) - a2 * a2 * (phx0 - phi0 - dphi0 * a1)) * div;
      const double cb = (-a1 * a1 * a1 * (phx1 - phi0 - dphi0 * a2) + a2 * a2 * a2 * (phx0 - phi0 - dphi0 * a1)) * div;
      if (fabs(ca) <= 1e-14 * fabs(cb) || ca == 0.0) at = dphi0 / (2.0 * cb);
      else { const double dd = std::max(cb * cb - 3.0 * ca * dphi0, 0.0); at = (-cb + sqrt(dd)) / (3.0 * ca); }
    }
    a1 = a2;
    at = std::min(at, a2 * rho_hi);
    a2 = std::max(at, a2 * rho_lo);
    phx0 = phx1;
    B200_TRY(phi(a2, &phx1));
  }
  *alpha = a2;
  return B200_OK;
}

// GenericTrustRegionScheme solve! (trust_region.jl:396-430, 511-513): the trial point u + du, the ratio rho of actual to
// predicted decrease, the radius update of the scheme (:431-520), then the step is taken or not.  dJJd = ||J du||^2 when the
// dogleg already has it.
static int32_t trust_region_step(b200_newton* nw, bool have_dJJd, double dJJd, int* accepted, double* objective, double* du_norm) {
  b200_ctx* ctx = nw->ctx;
  const int64_t n = nw->n;
  const TrParams& p = nw->trp;
  B200_TRY(trial_point(nw, 1.0, nw->du));
  CUDA_TRY(ctx, cudaMemsetAsync(ctx->d_scalars, 0, sizeof(double) * 2, ctx->stream));
  B200_TRY(b200i_residual_norm(nw->prob, nw->u_trial, nw->fu_trial, ctx->d_scalars));
  nw->res.nf += 1;
  // the six scalars of the acceptance test are independent: reduced on the device one after the other, fetched ONCE
  // (round 1 synchronised the host after each of them; VERDICT r1 weak #11)
  if (!have_dJJd) {
    B200_TRY(b200_jvp(nw->prob, nw->u, nw->du, nw->Jdu));
    B200_TRY(b200i_reduce_sum_dev(ctx, n, nw->Jdu, nw->Jdu, RED_DOT, ctx->d_scalars + 1));
  }
  B200_TRY(b200_vjp(nw->prob, nw->u, nw->fu, nw->JTfu));
  B200_TRY(b200i_reduce_sum_dev(ctx, n, nw->fu_trial, nullptr, RED_SUMSQ, ctx->d_scalars + 2));
  B200_TRY(b200i_reduce_sum_dev(ctx, n, nw->fu, nullptr, RED_SUMSQ, ctx->d_scalars + 3));
  B200_TRY(b200i_reduce_sum_dev(ctx, n, nw->du, nw->JTfu, RED_DOT, ctx->d_scalars + 4));
  B200_TRY(b200i_reduce_sum_dev(ctx, n, nw->du, nullptr, RED_SUMSQ, ctx->d_scalars + 5));
  B200_TRY(b200i_fetch_scalars(ctx, 6));
  const double trial_inf = ctx->h_scalars[0];
  if (!have_dJJd) dJJd = ctx->h_scalars[1];
  const double nt = sqrt(ctx->h_scalars[2]), nc = sqrt(ctx->h_scalars[3]), dg = ctx->h_scalars[4];
  const double num = (nt * nt - nc * nc) / 2.0;
  const double denom = dg + dJJd / 2.0;
  const double rho = num / denom;
  *accepted = rho > p.step_thr;
  const double dun = sqrt(ctx->h_scalars[5]);  // internalnorm(du)
  const int sch = nw->o.tr_scheme;
  double& tr = nw->trust_region;
  if (sch == B200_TR_SIMPLE) {  // trust_region.jl:431-440
    if (rho < p.shrink_thr) { tr *= p.shrink_fac; nw->shrink_counter += 1; }
    else { nw->shrink_counter = 0; if (rho > p.expand_thr && rho > p.step_thr) tr = p.expand_fac * tr; }
  } else if (sch == B200_TR_NLSOLVE) {  // :441-455
    if (rho < p.shrink_thr) { tr *= p.shrink_fac; nw->shrink_counter += 1; }
    else {
      nw->shrink_counter = 0;
      if (rho >= p.expand_thr) tr = p.expand_fac * dun;
      else if (rho >= nw->tp1) tr = std::max(tr, p.expand_fac * dun);
    }
  } else if (sch == B200_TR_NOCEDAL_WRIGHT) {  // :456-466
    if (rho < p.shrink_thr) { tr = p.shrink_fac * dun; nw->shrink_counter += 1; }
    else { nw->shrink_counter = 0; if (rho > p.expand_thr && fabs(dun - tr) < 1.0e-6 * tr) tr = p.expand_fac * tr; }
  } else if (sch == B200_TR_HEI) {  // :467-476, rfunc_adaptive_trust_region :383-391
    const double M = nw->tp1, g1 = nw->tp3, g2 = nw->tp4, beta = nw->tp2;
    const double rf = (rho >= p.shrink_thr) ? (2.0 * (M - 1.0 - g2) * atan(rho - p.shrink_thr) + (1.0 + g2)) / M_PI
                                            : (1.0 - g1 - beta) * (exp(rho - p.shrink_thr) + beta / (1.0 - g1 - beta));
    const double tr_new = rf * dun;
    if (tr_new < tr) nw->shrink_counter += 1; else nw->shrink_counter = 0;
    tr = tr_new;
  } else if (sch == B200_TR_YUAN) {  // :477-490
    if (rho < p.shrink_thr) { nw->tp1 = nw->tp2 * nw->tp1; nw->shrink_counter += 1; }
    else { if (rho >= p.expand_thr && 2.0 * dun > tr) nw->tp1 = nw->tp3 * nw->tp1; nw->shrink_counter = 0; }
    double g;
    B200_TRY(b200_vjp(nw->prob, nw->u_trial, nw->fu_trial, nw->JTfu));
    B200_TRY(h_nrm2(nw, nw->JTfu, &g));
    tr = nw->tp1 * g;
  } else if (sch == B200_TR_FAN) {  // :491-499
    if (rho < p.shrink_thr) { nw->tp1 *= nw->tp2; nw->shrink_counter += 1; }
    else { nw->shrink_counter = 0; if (rho > p.expand_thr) nw->tp1 = std::min(nw->tp1 * nw->tp3, nw->tp4); }
    tr = nw->tp1 * pow(nt, 0.99);
  } else if (sch == B200_TR_BASTIN) {  // :500-520, retrospective ratio at the trial point with the step just taken
    if (rho > p.step_thr) {
      double d1, d2;
      B200_TRY(b200_jvp(nw->prob, nw->u_trial, nw->du, nw->Jdu));
      B200_TRY(b200_vjp(nw->prob, nw->u_trial, nw->fu_trial, nw->JTfu));
      B200_TRY(h_dot(nw, nw->JTfu, nw->JTfu, &d1));
      B200_TRY(b200_vjp(nw->prob, nw->u_trial, nw->Jdu, nw->JTfu));
      B200_TRY(h_dot(nw, nw->JTfu, nw->JTfu, &d2));
      const double rho_retro = num / (d1 + d2 / 2.0);
      if (rho_retro >= p.expand_thr) tr = nw->tp1 * dun;
      nw->shrink_counter = 0;
    } else { tr *= nw->tp2; nw->shrink_counter += 1; }
  }
  tr = std::min(tr, nw->max_tr);
  if (*accepted) {
    accept_trial(nw);
    *objective = trial_inf;
    *du_norm = dun;
  } else {
    nw->make_new_jacobian = 0;
    *objective = nw->fnorm_inf;
    *du_norm = 0.0;
  }
  if (nw->shrink_counter > p.max_shrink) { nw->retcode = B200_RC_SHRINK_THRESHOLD_EXCEEDED; nw->force_stop = 1; }
  return B200_OK;
}

// step! (solve.jl:325-465): refresh J, solve, retry once with a fresh Jacobian, descend, globalise, end the step
static int32_t newton_step_inner(b200_newton* nw) {
  if (nw->o.descent == B200_DESCENT_LEVENBERG_MARQUARDT) return lm_step(nw);
  if (nw->o.descent == B200_DESCENT_BROYDEN) return broyden_step(nw);
  const b200_newton_opts& o = nw->o;
  bool fresh, ok;
  b200_gmres_stats gs;
  auto attempt = [&](bool first) -> int32_t {
    B200_TRY(refresh_jacobian(nw, &fresh));
    B200_TRY(pre_step(nw, first, fresh));
    return linear_solve(nw, fresh, &ok, &gs);
  };
  B200_TRY(attempt(true));
  if (!ok && !fresh) {  // solve.jl:367-382
    nw->make_new_jacobian = 1;
    B200_TRY(attempt(false));
  }
  if (!ok) { nw->retcode = B200_RC_INTERNAL_LINSOLVE_FAILED; nw->force_stop = 1; return B200_OK; }
  B200_TRY(b200_axpby(nw->ctx, nw->n, -1.0, nw->xlin, 0.0, nw->du));  // du = -x   (@. du *= -1, newton.jl:138)
  const bool tr_on = o.globalization == B200_GLOBALIZATION_TRUST_REGION;
  bool have_dJJd = false;
  double dJJd = 0.0;
  if (tr_on) B200_TRY(dogleg(nw, &have_dJJd, &dJJd));
  if (o.forcing == B200_FORCING_EW2 && krylov_linsolve(o)) {  // post_step_forcing!  eisenstat_walker.jl:83-87 (fu is still the old residual)
    nw->rnorm_prev = nw->rnorm;
    B200_TRY(h_nrm2(nw, nw->fu, &nw->rnorm));
  }
  nw->make_new_jacobian = 1;
  const bool ls_on = o.globalization == B200_GLOBALIZATION_LINESEARCH;
  int accepted = 1;
  double objective, du_norm, alpha = 1.0;
  if (ls_on) {
    B200_TRY(backtracking(nw, &alpha));
    B200_TRY(update_u(nw, alpha, &objective, &du_norm));  // @bb axpy!(alpha, du, u) ; evaluate_f!   solve.jl:403-407
  } else if (!tr_on) {  // solve.jl:436-445
    B200_TRY(update_u(nw, 1.0, &objective, &du_norm));
    nw->bytes += 5.0 * (8.0 * (double)nw->n);
  } else {
    B200_TRY(trust_region_step(nw, have_dJJd, dJJd, &accepted, &objective, &du_norm));
  }
  b200_trace_rec t = {};
  t.accepted = accepted; t.lin_iters = gs.iters; t.lin_status = gs.status; t.lin_rnorm = gs.rnorm;
  t.trust_radius = ls_on ? alpha : (o.descent == B200_DESCENT_PSEUDO_TRANSIENT) ? 1.0 / nw->alpha_inv : nw->trust_region;
  return step_end(nw, objective, du_norm, t);
}

// CommonSolve.step! (NonlinearSolveBase/src/solve.jl:835-858): one step, the counters, and the wall-clock limit
static int32_t newton_timed_step(b200_newton* nw) {
  const bool limited = nw->o.maxtime > 0.0;
  std::chrono::steady_clock::time_point t0;
  if (limited) t0 = std::chrono::steady_clock::now();
  B200_TRY(newton_step_inner(nw));
  nw->res.nsteps += 1;
  nw->nsteps += 1;
  if (limited) {
    CUDA_TRY(nw->ctx, cudaStreamSynchronize(nw->ctx->stream));
    nw->total_time += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    if (!nw->force_stop && nw->retcode == B200_RC_DEFAULT && nw->total_time >= nw->o.maxtime) { nw->retcode = B200_RC_MAXTIME; nw->force_stop = 1; }
  }
  return B200_OK;
}

int32_t b200_newton_step(b200_newton* nw, int32_t* terminated_host) {
  B200_DEVICE_GUARD(nw ? nw->ctx : nullptr);
  b200_ctx* ctx = nw->ctx;
  B200_REQUIRE(ctx, nw->initialised, "newton_step before newton_reinit");
  if (!(nw->force_stop || nw->nsteps >= nw->maxiters)) {  // not_terminated  abstract_types.jl:722-724
    B200_TRY(newton_timed_step(nw));
  }
  if (terminated_host) *terminated_host = (nw->force_stop || nw->nsteps >= nw->maxiters) ? 1 : 0;
  return B200_OK;
}

int32_t b200_newton_result_get(b200_newton* nw, b200_newton_result* r) {
  *r = nw->res;
  r->retcode = nw->retcode;
  r->resid_inf = nw->fnorm_inf;
  r->ntrace = (int32_t)nw->trace.size();
  r->bytes = nw->bytes;
  return B200_OK;
}

int32_t b200_newton_solve(b200_newton* nw, b200_newton_result* result) {
  B200_DEVICE_GUARD(nw ? nw->ctx : nullptr);
  b200_ctx* ctx = nw->ctx;
  B200_REQUIRE(ctx, nw->initialised, "newton_solve before newton_reinit");
  while (!nw->force_stop && nw->nsteps < nw->maxiters) B200_TRY(newton_timed_step(nw));
  if (nw->retcode == B200_RC_DEFAULT) nw->retcode = (nw->nsteps >= nw->maxiters) ? B200_RC_MAXITERS : B200_RC_SUCCESS;  // solve.jl:372-376
  // update_from_termination_cache! for Best modes: roll back to the best iterate (termination_conditions.jl:440-453)
  if (nw->best_u) {
    int32_t same = 1;
    B200_TRY(b200_equal(ctx, nw->n, nw->u, nw->best_u, &same));
    if (!same) {
      CUDA_TRY(ctx, cudaMemcpyAsync(nw->u, nw->best_u, sizeof(double) * nw->n, cudaMemcpyDeviceToDevice, ctx->stream));
      CUDA_TRY(ctx, cudaMemsetAsync(ctx->d_scalars, 0, sizeof(double), ctx->stream));
      B200_TRY(b200i_residual_norm(nw->prob, nw->u, nw->fu, ctx->d_scalars));
      nw->res.nf += 1;
      B200_TRY(b200i_fetch_scalars(ctx, 1));
      nw->fnorm_inf = ctx->h_scalars[0];
    }
  }
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (result) B200_TRY(b200_newton_result_get(nw, result));
  return B200_OK;
}

int32_t b200_newton_u(b200_newton* nw, double** u_dev) { *u_dev = nw->u; return B200_OK; }
int32_t b200_newton_fu(b200_newton* nw, double** fu_dev) { *fu_dev = nw->fu; return B200_OK; }

int32_t b200_newton_trace(b200_newton* nw, b200_trace_rec* recs, int32_t cap, int32_t* count) {
  int32_t m = (int32_t)std::min<size_t>(nw->trace.size(), (size_t)std::max(cap, 0));
  for (int32_t i = 0; i < m; ++i) recs[i] = nw->trace[i];
  if (count) *count = m;
  return B200_OK;
}

int32_t b200_newton_solve_host(b200_newton* nw, const double* u0_host, double* u_host, double* resid_host, b200_newton_result* result) {
  B200_DEVICE_GUARD(nw ? nw->ctx : nullptr);
  b200_ctx* ctx = nw->ctx;
  const size_t bytes = sizeof(double) * nw->n;
  CUDA_TRY(ctx, cudaMemcpyAsync(nw->u, u0_host, bytes, cudaMemcpyHostToDevice, ctx->stream));
  B200_TRY(b200_newton_reinit(nw, nw->u));
  B200_TRY(b200_newton_solve(nw, result));
  if (u_host) CUDA_TRY(ctx, cudaMemcpyAsync(u_host, nw->u, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  if (resid_host) CUDA_TRY(ctx, cudaMemcpyAsync(resid_host, nw->fu, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return B200_OK;
}
}  // extern "C"
