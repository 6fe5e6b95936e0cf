// mg.cu — geometric-multigrid V-cycle of the Brusselator Jacobian as a GMRES preconditioner (SURVEY.md §8f-2).
//
// Reference interface: LinearSolve `precs(A, p) -> (Pl, Pr)` on `KrylovJL_GMRES` (docs/src/tutorials/large_systems.md:244-316
// builds `AlgebraicMultigrid.ruge_stuben(W)` / `smoothed_aggregation(W)` and hands `aspreconditioner(...)` to GMRES;
// test/Core/core_tests__item21.jl).  On the structured periodic grid of the built-in problems the hierarchy is geometric:
//   * the grid of N points per dimension is coarsened by the prime factors of N, smallest first, down to ONE cell
//     (N = 100: 100 -> 50 -> 25 -> 5 -> 1), so the near-null space of the periodic Laplacian (constants per species) is
//     resolved exactly by the last level, a 2x2 solve with the mean reaction block;
//   * transfers for a factor r: vertex-centred multilinear interpolation and its scaled transpose (r = 2: full weighting);
//   * coarse operators are re-discretisations: a_c = a / r^2, reaction block from the restricted state;
//   * smoother: damped block-Jacobi on the 2x2 species blocks (omega = 0.8), nu pre + nu post sweeps, nu = 2 for r = 2
//     and 2 r for an odd factor r.
// One application (zero initial guess, fixed sweeps) is a fixed linear operator M^-1 ~ J(u)^-1: valid for left or right
// preconditioning of plain GMRES.  Everything is elementwise / stencil work on data that is tiny next to the Krylov basis:
// one kernel family (`mg_op_kernel`), HBM-bound, ~5 fine-grid stencil sweeps per application.
#include "common.cuh"
#include "mg_cell.cuh"
#include <math.h>
#include <vector>

namespace {
constexpr int MG_THREADS = 256;
constexpr int MG_MAX_LEVELS = 24;

struct MgLevel {
  int N, dim, ratio;     // points per dimension; coarsening ratio TO the next level (0 on the last level)
  int64_t NC;            // cells
  double a;              // Laplacian coefficient alpha / h^2 of this level
  double* state;         // 2 NC: (u, v) restricted to this level (level 0: borrowed pointer to the iterate)
  double *x, *x2, *b, *r;  // 2 NC each (level 0: b and the result are the caller's vectors)
};

// MODE 0: out = A x ; 1: out = b - A x ; 2: out = x + omega D^-1 (b - A x) ; 3: out = omega D^-1 b  (x == 0)
template <int MODE>
__global__ void __launch_bounds__(MG_THREADS) mg_op_kernel(int N, int dim, int64_t NC, double a, double A, const double* __restrict__ state,
                                                            const double* __restrict__ x, const double* __restrict__ b, double* __restrict__ out,
                                                            double omega) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= NC) return;
  mg_op_cell<MODE>(c, N, dim, NC, a, A, state, x, b, out, omega);
}

// Transfers (mg_cell.cuh): one thread per coarse (restrict) / fine (prolong) cell; the coarse grids are tiny next to the fine one.
__global__ void __launch_bounds__(MG_THREADS) mg_restrict_kernel(int Nf, int Nc, int dim, int ratio, const double* __restrict__ fine,
                                                                  double* __restrict__ coarse) {
  const int64_t NCc = dim == 3 ? (int64_t)Nc * Nc * Nc : (int64_t)Nc * Nc;
  const int64_t C = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (C >= NCc) return;
  mg_restrict_cell(C, Nf, Nc, dim, ratio, fine, coarse);
}

__global__ void __launch_bounds__(MG_THREADS) mg_prolong_add_kernel(int Nf, int Nc, int dim, int ratio, const double* __restrict__ coarse,
                                                                     double* __restrict__ fine) {
  const int64_t NCf = dim == 3 ? (int64_t)Nf * Nf * Nf : (int64_t)Nf * Nf;
  const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= NCf) return;
  mg_prolong_add_cell(f, Nf, Nc, dim, ratio, coarse, fine);
}

inline int mg_grid(int64_t n) { return (int)((n + MG_THREADS - 1) / MG_THREADS); }
}  // namespace

struct b200_mg {
  b200_ctx* ctx;
  const b200_problem* prob;  // the problem whose Jacobian this approximates: its A is read at every setup (b200_problem_set_AB)
  int dim, nlev;
  double A;                  // the reaction parameter of the current linearisation point
  double omega;
  MgLevel lev[MG_MAX_LEVELS];
  std::vector<double*> owned;
  // One application = ~60 launches on grids of 10^6 down to ONE cell: a few us of GPU time each (0.44 ms in all), but ~5 us of host
  // time to enqueue every one — a preconditioned solve was host-bound (5 100 launches per config-3 solve).  The V-cycle is captured once per
  // linearisation point into a CUDA graph (fixed input = lev[0].b, fixed result buffer) and replayed with one launch per application.
  cudaGraphExec_t gexec = nullptr;
  double* gres = nullptr;       // where the captured cycle leaves its result
  int64_t glaunches = 0;        // kernel launches inside the captured cycle (for the launch counter)
  bool graph_unavailable = false;
};

namespace {
int smallest_factor(int n) {
  for (int p = 2; (int64_t)p * p <= n; ++p)
    if (n % p == 0) return p;
  return n;
}

template <int MODE>
int32_t mg_op(b200_mg* mg, const MgLevel& L, const double* x, const double* b, double* out, double omega) {
  b200_ctx* ctx = mg->ctx;
  LAUNCH(ctx, (mg_op_kernel<MODE>), mg_grid(L.NC), MG_THREADS, 0, L.N, L.dim, L.NC, L.a, mg->A, (const double*)L.state, x, b, out, omega);
  CHECK_LAUNCH(ctx);
  return B200_OK;
}

// x_out = V-cycle(level l, b): result in *xres (one of the level's two iterate buffers, or `out0` on level 0)
int32_t mg_vcycle(b200_mg* mg, int l, const double* b, double** xres) {
  b200_ctx* ctx = mg->ctx;
  MgLevel& L = mg->lev[l];
  double* cur = L.x;
  double* nxt = L.x2;
  if (l == mg->nlev - 1) {  // one cell per species pair left (or no factor to coarsen by): exact block solve / plain smoothing
    B200_TRY(mg_op<3>(mg, L, nullptr, b, cur, L.N == 1 ? 1.0 : mg->omega));
    if (L.N > 1)  // a grid that cannot be coarsened (large prime N): smoothing only
      for (int s = 0; s < 7; ++s) { B200_TRY(mg_op<2>(mg, L, cur, b, nxt, mg->omega)); std::swap(cur, nxt); }
    *xres = cur;
    return B200_OK;
  }
  // nu pre + nu post sweeps: 2 for a coarsening by 2, 2 r for an odd ratio r (wavelengths up to 2 r h are the smoother's job)
  const int nu = L.ratio == 2 ? 2 : 2 * L.ratio;
  B200_TRY(mg_op<3>(mg, L, nullptr, b, cur, mg->omega));  // first pre-smoothing sweep from the zero guess
  for (int s = 1; s < nu; ++s) { B200_TRY(mg_op<2>(mg, L, cur, b, nxt, mg->omega)); std::swap(cur, nxt); }
  B200_TRY(mg_op<1>(mg, L, cur, b, L.r, 0.0));
  MgLevel& Cl = mg->lev[l + 1];
  LAUNCH(ctx, mg_restrict_kernel, mg_grid(Cl.NC), MG_THREADS, 0, L.N, Cl.N, L.dim, L.ratio, (const double*)L.r, Cl.b);
  double* xc = nullptr;
  B200_TRY(mg_vcycle(mg, l + 1, Cl.b, &xc));
  LAUNCH(ctx, mg_prolong_add_kernel, mg_grid(L.NC), MG_THREADS, 0, L.N, Cl.N, L.dim, L.ratio, (const double*)xc, cur);
  CHECK_LAUNCH(ctx);
  for (int s = 0; s < nu; ++s) { B200_TRY(mg_op<2>(mg, L, cur, b, nxt, mg->omega)); std::swap(cur, nxt); }
  *xres = cur;
  return B200_OK;
}
}  // namespace

// ---- internal API used by the linear-operator layer (gmres.cu) and the Newton driver
int32_t b200i_mg_create(b200_problem* prob, b200_mg** out) {
  b200_ctx* ctx = prob->ctx;
  B200_REQUIRE(ctx, prob->kind == B200_PROB_BRUSS2D || prob->kind == B200_PROB_BRUSS3D, "multigrid preconditioner: built-in Brusselator problems only");
  b200_mg* mg = new b200_mg();
  mg->ctx = ctx; mg->prob = prob; mg->dim = prob->kind == B200_PROB_BRUSS3D ? 3 : 2; mg->A = prob->A; mg->omega = 0.8; mg->nlev = 0;
  int N = prob->N;
  double a = prob->a;
  for (;;) {
    MgLevel& L = mg->lev[mg->nlev];
    L.N = N; L.dim = mg->dim; L.a = a;
    L.NC = mg->dim == 3 ? (int64_t)N * N * N : (int64_t)N * N;
    L.ratio = (N > 1 && mg->nlev + 1 < MG_MAX_LEVELS) ? smallest_factor(N) : 0;
    // a prime N > 3 cannot be coarsened geometrically: it goes straight to the one-cell level through one aggregation step
    // only while that stays cheap (block of N^dim cells per coarse cell); otherwise the hierarchy ends here (smoothing only)
    if (L.ratio > 7 && L.ratio == N && L.NC > 4096) L.ratio = 0;
    L.state = L.x = L.x2 = L.b = L.r = nullptr;
    double** bufs[] = {&L.x, &L.x2, &L.b, &L.r, &L.state};
    for (int q = 0; q < 5; ++q) {
      if (mg->nlev == 0 && q == 4) break;  // level 0 borrows the iterate
      if (cudaMalloc(bufs[q], sizeof(double) * 2 * L.NC) != cudaSuccess) {
        cudaGetLastError();
        for (double* p : mg->owned) cudaFree(p);
        delete mg;
        return ctx->fail(B200_ERR_NOMEM, "multigrid preconditioner: out of device memory", __FILE__, __LINE__);
      }
      mg->owned.push_back(*bufs[q]);
    }
    mg->nlev += 1;
    if (L.ratio == 0) break;
    N /= L.ratio;
    a /= (double)L.ratio * L.ratio;
  }
  *out = mg;
  return B200_OK;
}

int32_t b200i_mg_destroy(b200_mg* mg) {
  if (!mg) return B200_OK;
  cudaStreamSynchronize(mg->ctx->stream);
  if (mg->gexec) cudaGraphExecDestroy(mg->gexec);
  for (double* p : mg->owned) cudaFree(p);
  delete mg;
  return B200_OK;
}

// (re)build the coarse operators for the linearisation point u: restrict the state level by level (the same transfer as the
// residuals), a_l is fixed by the geometry, A is the problem's current one (it changes under b200_problem_set_AB: reinit with new
// parameters, or the ensemble's per-trajectory route).  Called once per Newton step, like update_A! rebuilds Pl / Pr.
int32_t b200i_mg_setup(b200_mg* mg, const double* u) {
  b200_ctx* ctx = mg->ctx;
  mg->A = mg->prob->A;
  mg->lev[0].state = const_cast<double*>(u);
  for (int l = 0; l + 1 < mg->nlev; ++l) {
    MgLevel &L = mg->lev[l], &Cl = mg->lev[l + 1];
    LAUNCH(ctx, mg_restrict_kernel, mg_grid(Cl.NC), MG_THREADS, 0, L.N, Cl.N, L.dim, L.ratio, (const double*)L.state, Cl.state);
  }
  CHECK_LAUNCH(ctx);
  // the captured cycle has the level states' addresses and values baked in as of its capture: a new linearisation point needs a new one
  if (mg->gexec) { CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream)); cudaGraphExecDestroy(mg->gexec); mg->gexec = nullptr; }
  return B200_OK;
}

int32_t b200i_mg_apply(b200_mg* mg, const double* x, double* y) {
  b200_ctx* ctx = mg->ctx;
  const size_t bytes = sizeof(double) * 2 * mg->lev[0].NC;
  if (!mg->gexec && !mg->graph_unavailable && !ctx->prof_on) {
    cudaGraph_t graph = nullptr;
    const int64_t l0 = ctx->launches;
    double* res = nullptr;
    if (cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
      const int32_t rc = mg_vcycle(mg, 0, mg->lev[0].b, &res);
      const cudaError_t e = cudaStreamEndCapture(ctx->stream, &graph);
      if (rc == B200_OK && e == cudaSuccess && graph && cudaGraphInstantiate(&mg->gexec, graph, 0) == cudaSuccess) {
        mg->gres = res;
        mg->glaunches = ctx->launches - l0;
      } else {
        mg->gexec = nullptr;
        mg->graph_unavailable = true;
        cudaGetLastError();
      }
      if (graph) cudaGraphDestroy(graph);
      ctx->launches = l0;  // nothing ran yet
    } else {
      mg->graph_unavailable = true;
      cudaGetLastError();
    }
  }
  if (mg->gexec) {
    CUDA_TRY(ctx, cudaMemcpyAsync(mg->lev[0].b, x, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
    CUDA_TRY(ctx, cudaGraphLaunch(mg->gexec, ctx->stream));
    ctx->launches += mg->glaunches;
    CUDA_TRY(ctx, cudaMemcpyAsync(y, mg->gres, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
    return B200_OK;
  }
  double* res = nullptr;
  B200_TRY(mg_vcycle(mg, 0, x, &res));
  CUDA_TRY(ctx, cudaMemcpyAsync(y, res, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
  return B200_OK;
}

int32_t b200i_mg_levels(b200_mg* mg, int32_t* nlev, int32_t* sizes, int32_t cap) {
  *nlev = mg->nlev;
  for (int l = 0; l < mg->nlev && l < cap; ++l) sizes[l] = mg->lev[l].N;
  return B200_OK;
}
