// ensemble.cu — K independent 2D Brusselator solves (SURVEY.md §8a row a11, config 5).
//
// Semantics: SciMLBase EnsembleProblem as used at test/PolyAlgorithms/core_tests__item6.jl:3-20 — trajectory m is an
// ordinary NewtonRaphson solve of `remake(prob; p = (A_m, B_m, alpha, dx), u0 = u0[:, m])`, no shared state, results
// collected in order.  Sharding across GPUs is done by the caller (one rank per GPU, contiguous trajectory blocks);
// this file is the per-GPU batch.
//
// Two engines:
//   * batched (N <= 32): one CTA per trajectory, persistent over a work queue; iterate, residual, Krylov direction and the
//     Givens recurrence live in shared memory, the Krylov basis streams through a per-CTA slab in HBM/L2; with
//     Multigrid("left" / "right") the whole V-cycle hierarchy lives in shared memory too; TrustRegion (Dogleg) and
//     BackTracking without a preconditioner globalise each step inside the same kernel (see ens_batched.cu)
//   * sequential fallback (any N): the single-system driver of newton.cu, one trajectory after another (block-Jacobi and
//     every option set the batched kernel does not cover).
#include "common.cuh"
#include <algorithm>
#include <vector>

int32_t b200i_ens_batched_supported(int32_t N, const b200_newton_opts* o);
int32_t b200i_ens_batched_solve(b200_ctx* ctx, int32_t N, int32_t nprob, double alpha, const b200_newton_opts* o, const double* u0,
                                const double* A, const double* B, double* u_out, double* resid_inf, int32_t* retcodes, int32_t* nsteps,
                                int32_t* njvp, void** workspace, size_t* workspace_bytes, int32_t* n_deferred);
int32_t b200i_ens_batched_ctas_per_sm(b200_ctx* ctx, int32_t N, const b200_newton_opts* o, int32_t* per_sm);
int32_t b200i_ens_batched_precond_apply(b200_ctx* ctx, int32_t N, int32_t nprob, double alpha, const b200_newton_opts* o, const double* u,
                                        const double* A, const double* x, double* y);

struct b200_ensemble {
  b200_ctx* ctx;
  int32_t N, nprob;
  double alpha;
  b200_newton_opts o;
  int32_t batched;     // the one-CTA-per-trajectory kernel covers this option set
  b200_problem* prob;  // sequential engine (whole ensemble when !batched; deferred trajectories otherwise, created on first use)
  b200_newton* nw;
  void* workspace;     // batched engine
  size_t workspace_bytes;
  int32_t *d_rc, *d_ns, *d_nj;
  double* d_res;
};

namespace {
__global__ void ens_store_kernel(int32_t m, double resid, int32_t rc, int32_t ns, int32_t nj, double* resid_inf, int32_t* retcodes,
                                 int32_t* nsteps, int32_t* njvp) {
  if (resid_inf) resid_inf[m] = resid;
  if (retcodes) retcodes[m] = rc;
  if (nsteps) nsteps[m] = ns;
  if (njvp) njvp[m] = nj;
}
}  // namespace

extern "C" {
int32_t b200_ens_destroy(b200_ensemble* e) {
  B200_DEVICE_GUARD(e ? e->ctx : nullptr);
  if (!e) return B200_OK;
  cudaStreamSynchronize(e->ctx->stream);
  if (e->nw) b200_newton_destroy(e->nw);
  if (e->prob) b200_problem_destroy(e->prob);
  if (e->workspace) cudaFree(e->workspace);
  cudaFree(e->d_rc); cudaFree(e->d_ns); cudaFree(e->d_nj); cudaFree(e->d_res);
  delete e;
  return B200_OK;
}

int32_t b200_ens_create(b200_ctx* ctx, int32_t N, int32_t nprob_local, double alpha, const b200_newton_opts* opts, b200_ensemble** out) {
  B200_DEVICE_GUARD(ctx);
  B200_REQUIRE(ctx, N >= 3 && nprob_local > 0 && opts && out, "ens_create: bad arguments");
  B200_REQUIRE(ctx, opts->linsolve == B200_LINSOLVE_GMRES && opts->descent == B200_DESCENT_NEWTON,
               "ensemble: only matrix-free Newton(linsolve = GMRES) trajectories are batched: NewtonRaphson, with or without "
               "linesearch = BackTracking(), or TrustRegion");
  B200_REQUIRE(ctx, opts->globalization == B200_GLOBALIZATION_NONE || opts->globalization == B200_GLOBALIZATION_TRUST_REGION ||
                        opts->globalization == B200_GLOBALIZATION_LINESEARCH,
               "ensemble: unknown globalization");
  const int32_t pc = opts->precond;
  B200_REQUIRE(ctx, opts->globalization == B200_GLOBALIZATION_NONE || pc == B200_PRECOND_NONE,
               "ensemble: a globalised ensemble (TrustRegion, BackTracking) takes no preconditioner");
  B200_REQUIRE(ctx, pc != B200_PRECOND_ILU0_LEFT && pc != B200_PRECOND_ILU0_RIGHT && pc != B200_PRECOND_AMG_LEFT && pc != B200_PRECOND_AMG_RIGHT &&
                        pc != B200_PRECOND_SA_AMG_LEFT && pc != B200_PRECOND_SA_AMG_RIGHT,
               "ensemble: ILU0 and AMG precondition the assembled sparse Jacobian, and ensemble trajectories are matrix-free: use "
               "Multigrid or BlockJacobi");
  B200_REQUIRE(ctx, pc == B200_PRECOND_NONE || pc == B200_PRECOND_BLOCK_JACOBI_LEFT || pc == B200_PRECOND_BLOCK_JACOBI_RIGHT ||
                        pc == B200_PRECOND_MULTIGRID_LEFT || pc == B200_PRECOND_MULTIGRID_RIGHT,
               "ensemble: unknown preconditioner");
  b200_ensemble* e = new b200_ensemble();
  memset(e, 0, sizeof(*e));
  e->ctx = ctx; e->N = N; e->nprob = nprob_local; e->alpha = alpha; e->o = *opts;
  e->o.store_trace = 0;
  CUDA_TRY(ctx, cudaMalloc(&e->d_rc, sizeof(int32_t) * nprob_local));
  CUDA_TRY(ctx, cudaMalloc(&e->d_ns, sizeof(int32_t) * nprob_local));
  CUDA_TRY(ctx, cudaMalloc(&e->d_nj, sizeof(int32_t) * nprob_local));
  CUDA_TRY(ctx, cudaMalloc(&e->d_res, sizeof(double) * nprob_local));
  e->batched = b200i_ens_batched_supported(N, &e->o);
  if (!e->batched) {
    int32_t s = b200_problem_create_bruss2d(ctx, N, 3.4, 1.0, alpha, &e->prob);
    if (s == B200_OK) s = b200_newton_create(e->prob, &e->o, &e->nw);
    if (s != B200_OK) { b200_ens_destroy(e); return s; }
  }
  *out = e;
  return B200_OK;
}

int32_t b200_ens_solve(b200_ensemble* e, const double* u0, const double* A, const double* B, double* u_out, double* resid_inf,
                       int32_t* retcodes, int32_t* nsteps, int32_t* njvp, b200_ens_result* result) {
  B200_DEVICE_GUARD(e ? e->ctx : nullptr);
  b200_ctx* ctx = e->ctx;
  const int64_t n = 2 * (int64_t)e->N * e->N;
  const int32_t K = e->nprob;
  B200_REQUIRE(ctx, u0 && A && B && u_out, "ens_solve: bad arguments");
  double* d_res = resid_inf ? resid_inf : e->d_res;
  int32_t* d_rc = retcodes ? retcodes : e->d_rc;
  int32_t* d_ns = nsteps ? nsteps : e->d_ns;
  int32_t* d_nj = njvp ? njvp : e->d_nj;
  // one trajectory through the general driver (remake(prob; p = ...), reinit, solve): the route for option sets the batched
  // kernel does not cover, and for trajectories whose Krylov basis outgrew the batched kernel's per-CTA slab
  auto solve_one = [&](int32_t m, double Am, double Bm) -> int32_t {
    B200_TRY(b200_problem_set_AB(e->prob, Am, Bm));
    B200_TRY(b200_newton_reinit(e->nw, u0 + (int64_t)m * n));
    b200_newton_result r;
    B200_TRY(b200_newton_solve(e->nw, &r));
    double* u;
    B200_TRY(b200_newton_u(e->nw, &u));
    CUDA_TRY(ctx, cudaMemcpyAsync(u_out + (int64_t)m * n, u, sizeof(double) * n, cudaMemcpyDeviceToDevice, ctx->stream));
    LAUNCH(ctx, ens_store_kernel, 1, 1, 0, m, r.resid_inf, r.retcode, r.nsteps, r.njvp, d_res, d_rc, d_ns, d_nj);
    CHECK_LAUNCH(ctx);
    return B200_OK;
  };
  std::vector<double> hA, hB;
  auto fetch_AB = [&]() -> int32_t {
    hA.resize(K); hB.resize(K);
    B200_TRY(b200_memcpy_d2h(ctx, hA.data(), A, sizeof(double) * K));
    B200_TRY(b200_memcpy_d2h(ctx, hB.data(), B, sizeof(double) * K));
    return B200_OK;
  };
  if (e->batched) {
    int32_t deferred = 0;
    B200_TRY(b200i_ens_batched_solve(ctx, e->N, K, e->alpha, &e->o, u0, A, B, u_out, d_res, d_rc, d_ns, d_nj, &e->workspace,
                                     &e->workspace_bytes, &deferred));
    if (deferred > 0) {
      if (!e->nw) {
        B200_TRY(b200_problem_create_bruss2d(ctx, e->N, 3.4, 1.0, e->alpha, &e->prob));
        B200_TRY(b200_newton_create(e->prob, &e->o, &e->nw));
      }
      std::vector<int32_t> hrc(K);
      B200_TRY(b200_memcpy_d2h(ctx, hrc.data(), d_rc, sizeof(int32_t) * K));
      B200_TRY(fetch_AB());
      for (int32_t m = 0; m < K; ++m)
        if (hrc[m] == B200I_ENS_RC_DEFERRED) B200_TRY(solve_one(m, hA[m], hB[m]));
    }
  } else {
    B200_TRY(fetch_AB());
    for (int32_t m = 0; m < K; ++m) B200_TRY(solve_one(m, hA[m], hB[m]));
  }
  if (result) {
    std::vector<double> hres(K);
    std::vector<int32_t> hrc(K), hns(K), hnj(K);
    B200_TRY(b200_memcpy_d2h(ctx, hres.data(), d_res, sizeof(double) * K));
    B200_TRY(b200_memcpy_d2h(ctx, hrc.data(), d_rc, sizeof(int32_t) * K));
    B200_TRY(b200_memcpy_d2h(ctx, hns.data(), d_ns, sizeof(int32_t) * K));
    B200_TRY(b200_memcpy_d2h(ctx, hnj.data(), d_nj, sizeof(int32_t) * K));
    memset(result, 0, sizeof(*result));
    result->nprob = K;
    for (int32_t m = 0; m < K; ++m) {
      if (hrc[m] == B200_RC_SUCCESS) result->nsuccess += 1;
      result->max_nsteps = std::max(result->max_nsteps, hns[m]);
      result->total_nsteps += hns[m];
      result->total_njvp += hnj[m];
      if (hres[m] > result->worst_resid_inf || hres[m] != hres[m]) result->worst_resid_inf = hres[m];
    }
  } else {
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  }
  return B200_OK;
}

int32_t b200_ens_precond_apply(b200_ensemble* e, const double* u_dev, const double* A_dev, const double* x_dev, double* y_dev) {
  B200_DEVICE_GUARD(e ? e->ctx : nullptr);
  if (!e) return B200_ERR_INVALID;
  b200_ctx* ctx = e->ctx;
  B200_REQUIRE(ctx, u_dev && A_dev && x_dev && y_dev, "ens_precond_apply: bad arguments");
  B200_REQUIRE(ctx, e->batched && (e->o.precond == B200_PRECOND_MULTIGRID_LEFT || e->o.precond == B200_PRECOND_MULTIGRID_RIGHT),
               "ens_precond_apply: only a batched multigrid ensemble applies its preconditioner");
  B200_TRY(b200i_ens_batched_precond_apply(ctx, e->N, e->nprob, e->alpha, &e->o, u_dev, A_dev, x_dev, y_dev));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return B200_OK;
}

int32_t b200_ens_ctas_per_sm(b200_ensemble* e, int32_t* ctas_per_sm) {
  B200_DEVICE_GUARD(e ? e->ctx : nullptr);
  if (!e) return B200_ERR_INVALID;
  B200_REQUIRE(e->ctx, ctas_per_sm, "ens_ctas_per_sm: bad arguments");
  *ctas_per_sm = 0;
  if (e->batched) B200_TRY(b200i_ens_batched_ctas_per_sm(e->ctx, e->N, &e->o, ctas_per_sm));
  return B200_OK;
}
}  // extern "C"
