// common.cuh — internal declarations shared by the translation units of libb200newton.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <vector>
#include "../../include/b200newton.h"

struct b200_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  int sm_count = 132;
  size_t smem_optin = 0;
  size_t l2_bytes = 0;
  std::string last_error;
  int64_t launches = 0;
  // reduction scratch: per-block partials + a few device scalars mirrored to pinned host memory
  double* d_partials = nullptr;  // RED_MAX_BLOCKS * 4 doubles
  double* d_scalars = nullptr;   // 64 doubles
  double* h_scalars = nullptr;   // pinned, 64 doubles
  void* l2_flush = nullptr;
  size_t l2_flush_bytes = 0;
  cudaStream_t aux_stream = nullptr;  // look-ahead panel factorisation of the dense LU
  cudaEvent_t ev_a = nullptr, ev_b = nullptr;
  unsigned long long* d_lu_xchg = nullptr;  // dense LU panel: flag-in-word exchange tables (dense.cu PX_WORDS)
  // optional per-kernel-family event timing (b200_ctx_profile_*)
  bool prof_on = false;
  struct ProfSlot { double ms = 0, bytes = 0; int64_t launches = 0; } prof[B200_KID_COUNT];
  struct ProfPending { int kid; double bytes; cudaEvent_t a, b; };
  std::vector<ProfPending> prof_pending;
  std::vector<cudaEvent_t> prof_free;
  void prof_begin(int kid, double bytes);
  void prof_end();
  void prof_collect();
  int32_t fail(int32_t code, const char* what, const char* file, int line);
};

// timed launch: like LAUNCH, bracketed by events when profiling is on
#define PLAUNCH(ctx, kid, bytes, kernel, grid, block, smem, ...)                        \
  do {                                                                                  \
    if ((ctx)->prof_on) (ctx)->prof_begin((kid), (bytes));                              \
    kernel<<<(grid), (block), (smem), (ctx)->stream>>>(__VA_ARGS__);                    \
    (ctx)->launches++;                                                                  \
    if ((ctx)->prof_on) (ctx)->prof_end();                                              \
  } while (0)

// Every extern "C" entry that takes a context or a handle makes the context's device current first: allocations, kernel
// launches and event records below it otherwise land on whichever device the calling thread used last (one process may hold
// contexts on several GPUs; api.default_context(device), a Julia host with one task per device).  Not restored on return.
#define B200_DEVICE_GUARD(ctxexpr)                                                      \
  do {                                                                                  \
    const b200_ctx* g__ = (ctxexpr);                                                    \
    int d__ = -1;                                                                       \
    if (g__ && (cudaGetDevice(&d__) != cudaSuccess || d__ != g__->device)) cudaSetDevice(g__->device); \
  } while (0)

#define B200_RED_MAX_BLOCKS 2048
enum { RED_DOT = 0, RED_SUMSQ = 1, RED_MAXABS = 2, RED_DIFFSQ = 3, RED_MIN = 4, RED_MAX = 5, RED_NEQ = 6,
       RED_SUMSQ2 = 7 /* sum (x+y)^2 */, RED_MAXABS2 = 8 /* max |x+y| */, RED_RELVIOL = 9 /* #{ |x| > a |x+y| } */,
       RED_COUNT_LE = 10 /* #{ |x| <= a } */, RED_COUNT_DIFF_LE = 11 /* #{ |x - y| <= a } */ };

#define CUDA_TRY(ctx, expr)                                                             \
  do {                                                                                  \
    cudaError_t e__ = (expr);                                                           \
    if (e__ != cudaSuccess) {                                                           \
      char buf__[512];                                                                  \
      snprintf(buf__, sizeof(buf__), "%s -> %s", #expr, cudaGetErrorString(e__));       \
      return (ctx)->fail(B200_ERR_CUDA, buf__, __FILE__, __LINE__);                     \
    }                                                                                   \
  } while (0)

#define B200_TRY(expr)                  \
  do {                                  \
    int32_t s__ = (expr);               \
    if (s__ != B200_OK) return s__;     \
  } while (0)

#define B200_REQUIRE(ctx, cond, msg)                                                    \
  do {                                                                                  \
    if (!(cond)) return (ctx)->fail(B200_ERR_INVALID, msg, __FILE__, __LINE__);         \
  } while (0)

// Every kernel launch goes through this so that b200_ctx_kernel_launches() is an honest count.
#define LAUNCH(ctx, kernel, grid, block, smem, ...)                                     \
  do {                                                                                  \
    kernel<<<(grid), (block), (smem), (ctx)->stream>>>(__VA_ARGS__);                    \
    (ctx)->launches++;                                                                  \
  } while (0)

#define CHECK_LAUNCH(ctx) CUDA_TRY(ctx, cudaPeekAtLastError())

// cooperative launch (every CTA co-resident, the guarantee of cudaLaunchCooperativeKernel), counted and timed like PLAUNCH
template <typename... Params, typename... Args>
int32_t coop_launch(b200_ctx* ctx, int kid, double bytes, void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, Args... args) {
  cudaLaunchAttribute coop;
  coop.id = cudaLaunchAttributeCooperative;
  coop.val.cooperative = 1;
  const cudaLaunchConfig_t cfg = {grid, block, smem, ctx->stream, &coop, 1};
  if (ctx->prof_on) ctx->prof_begin(kid, bytes);
  CUDA_TRY(ctx, cudaLaunchKernelEx(&cfg, kernel, args...));
  ctx->launches++;
  if (ctx->prof_on) ctx->prof_end();
  return B200_OK;
}

// ---------------------------------------------------------------- device helpers
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_min(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// block-wide sum; result valid in thread 0 (and warp 0). `red` must hold >= 32 doubles of shared memory.
__device__ __forceinline__ double block_sum(double v, double* red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[wid] = v;
  __syncthreads();
  v = (threadIdx.x < nw) ? red[threadIdx.x] : 0.0;
  if (wid == 0) v = warp_sum(v);
  return v;
}
__device__ __forceinline__ double block_max(double v, double* red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) red[wid] = v;
  __syncthreads();
  v = (threadIdx.x < nw) ? red[threadIdx.x] : 0.0;
  if (wid == 0) v = warp_max(v);
  return v;
}
// |x| with non-finite values mapped to +inf so that a max-reduction propagates them (Julia's maximum(abs, x) yields NaN;
// both are "non-finite" to the termination test at termination_conditions.jl:256).
__device__ __forceinline__ double abs_nf(double x) {
  double a = fabs(x);
  return (a == a) ? a : __longlong_as_double(0x7ff0000000000000LL);
}
__device__ __forceinline__ void atomic_max_nonneg(double* addr, double v) {  // v >= 0 or +inf: bit patterns are ordered
  atomicMax(reinterpret_cast<unsigned long long*>(addr), static_cast<unsigned long long>(__double_as_longlong(v)));
}

// ---------------------------------------------------------------- internal structs
struct b200_problem {
  b200_ctx* ctx;
  int32_t kind;
  int32_t N;
  int64_t n;
  double A, B, alpha, a;  // a = alpha / dx^2
  double p;
  const double* pvec;  // device
  b200_residual_cb f_cb;
  b200_jvp_cb jvp_cb, vjp_cb;
  b200_jac_cb jac_dense_cb, jac_nzval_cb;  // optional user jac! (b3)
  void* user;
  double* fd_scratch;  // n doubles, lazily allocated (callback finite differences)
  int64_t *proto_colptr, *proto_rowval;  // host copy (0-based) of a user jac_prototype pattern, or null
};

struct b200_sparse_jac;
struct b200_mg;

// ---- mbarrier + TMA bulk copy (cp.async.bulk, 1-D): a single thread starts a copy of `bytes` (multiple of 16, both addresses
//      16-byte aligned) that completes on an mbarrier; waits are bounded so a fault cannot hang the GPU
__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"((unsigned)__cvta_generic_to_shared(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(bytes) : "memory");
}
// gives up after 2^26 polls; sets *err (when given) so that the caller reports the timeout instead of using stale data
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned parity, int* err = nullptr) {
  const unsigned a = (unsigned)__cvta_generic_to_shared(bar);
  unsigned done = 0, spins = 0;
  while (!done) {
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(done) : "r"(a), "r"(parity) : "memory");
    if (++spins > (1u << 26)) {
      if (err) *err = 1;
      break;
    }
  }
}
__device__ __forceinline__ void tma_bulk_load(void* smem_dst, const void* gsrc, unsigned bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"((unsigned)__cvta_generic_to_shared(bar))
               : "memory");
}
// L2 cache policy for data read once: the lines an access with this hint touches are the first candidates for eviction, so
// streamed data does not push out what was prefetched into L2 for later.  Created at the point of use (one instruction) so
// that no register holds it across a loop.
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
// tma_bulk_load with an L2 cache policy (l2_evict_first_policy)
__device__ __forceinline__ void tma_bulk_load(void* smem_dst, const void* gsrc, unsigned bytes, uint64_t* bar, uint64_t policy) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
               ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gsrc), "r"(bytes), "r"((unsigned)__cvta_generic_to_shared(bar)), "l"(policy)
               : "memory");
}
// bulk prefetch of `bytes` (multiple of 16, 16-byte aligned) of global memory into L2; no completion to wait for
__device__ __forceinline__ void l2_bulk_prefetch(const void* gsrc, unsigned bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gsrc), "r"(bytes) : "memory");
}
// 16-byte global -> shared copy (non-bulk cp.async, L2 only); completes into the thread's current cp.async group
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
// the same with an L2 cache policy (l2_evict_first_policy)
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, uint64_t policy) {
  asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gsrc), "l"(policy)
               : "memory");
}
// orders this thread's generic-proxy accesses to shared memory (loads, stores, completed non-bulk cp.async) before later
// async-proxy (TMA) accesses; place it before the barrier after which one thread issues the bulk copy
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- flag-in-word cross-CTA exchange (the idea of NCCL's LL protocol): a 64-bit value travels as two 64-bit words of
//      {32 data bits | 32-bit epoch << 32}, written by ONE 16-byte store, so a reader that sees the expected epoch in both words
//      has the value — no fence, no atomic, no separate barrier, one L2 round trip.  The resident Arnoldi kernel (gmres.cu)
//      publishes with ll_store; the cooperative LU panel (dense.cu) uses all four parts.
__device__ __forceinline__ void ll_store(unsigned long long* dst, unsigned long long v, unsigned epoch) {
  const unsigned long long e = (unsigned long long)epoch << 32;
  asm volatile("st.relaxed.gpu.global.v2.u64 [%0], {%1, %2};" ::"l"(dst), "l"((v & 0xffffffffull) | e), "l"((v >> 32) | e) : "memory");
}
__device__ __forceinline__ ulonglong2 ll_load(const unsigned long long* src) {
  ulonglong2 p;
  asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(p.x), "=l"(p.y) : "l"(src) : "memory");
  return p;
}
// reload `p` from `src` until both words carry `epoch`; bounded so that a fault cannot hang the device: after `bound` reloads
// *fault = 1 and `p` is left as last read
__device__ __forceinline__ void ll_wait(const unsigned long long* src, ulonglong2& p, unsigned epoch, unsigned bound, int* fault) {
  unsigned spins = 0;
  while ((unsigned)(p.x >> 32) != epoch || (unsigned)(p.y >> 32) != epoch) {
    if (++spins > bound) { *fault = 1; break; }
    p = ll_load(src);
  }
}
__device__ __forceinline__ unsigned long long ll_value(ulonglong2 p) { return (p.x & 0xffffffffull) | (p.y << 32); }


constexpr int32_t B200I_ENS_RC_DEFERRED = -7;  // batched ensemble kernel -> host: redo this trajectory through the general driver (never returned to a caller)

// The radius update scheme's constants (get_parameters, trust_region.jl:348-381): thresholds, factors and the shrink limit
// hold for the solver's life; tp1..tp4 are the initial scheme parameters, restored by every reinit (Yuan and Fan mutate p1).
// Shared by the single-system driver (newton.cu) and the batched ensemble kernel (ens_batched.cu).
struct TrParams {
  double step_thr, shrink_thr, expand_thr, shrink_fac, expand_fac;
  int max_shrink;
  double tp1, tp2, tp3, tp4;
};
static inline TrParams b200i_tr_params(const b200_newton_opts& o) {
  const int sch = o.tr_scheme;
  TrParams p;
  p.step_thr = o.tr_step_threshold > 0 ? o.tr_step_threshold : (sch == B200_TR_HEI ? 0.0 : sch == B200_TR_YUAN ? 1.0 / 1000 : sch == B200_TR_BASTIN ? 1.0 / 20 : 1.0 / 10000);
  p.shrink_thr = o.tr_shrink_threshold > 0 ? o.tr_shrink_threshold : (sch == B200_TR_HEI ? 0.0 : (sch == B200_TR_NLSOLVE || sch == B200_TR_BASTIN) ? 1.0 / 20 : 0.25);
  p.expand_thr = o.tr_expand_threshold > 0 ? o.tr_expand_threshold : ((sch == B200_TR_NLSOLVE || sch == B200_TR_BASTIN) ? 0.9 : sch == B200_TR_HEI ? 0.0 : 0.75);
  p.shrink_fac = o.tr_shrink_factor > 0 ? o.tr_shrink_factor : (sch == B200_TR_NLSOLVE ? 0.5 : sch == B200_TR_HEI ? 0.0 : sch == B200_TR_BASTIN ? 1.0 / 20 : 0.25);
  p.expand_fac = o.tr_expand_factor > 0 ? o.tr_expand_factor : 2.0;
  p.max_shrink = o.max_shrink_times > 0 ? o.max_shrink_times : 32;
  p.tp1 = p.tp2 = p.tp3 = p.tp4 = 0.0;
  if (sch == B200_TR_NLSOLVE) { p.tp1 = 0.5; }
  else if (sch == B200_TR_HEI) { p.tp1 = 5.0; p.tp2 = 0.1; p.tp3 = 0.15; p.tp4 = 0.15; }
  else if (sch == B200_TR_YUAN) { p.tp1 = 2.0; p.tp2 = 1.0 / 6; p.tp3 = 6.0; }
  else if (sch == B200_TR_FAN) { p.tp1 = 0.1; p.tp2 = 0.25; p.tp3 = 12.0; p.tp4 = 1.0e18; }
  else if (sch == B200_TR_BASTIN) { p.tp1 = 2.5; p.tp2 = 0.25; }
  return p;
}

struct b200_linop {
  b200_ctx* ctx;
  int32_t kind;  // LINOP_*
  int64_t n;
  b200_problem* prob;
  const double* u;
  int32_t jvp_mode;
  const int64_t *colptr, *rowval;
  const double* nzval;
  int32_t index_base;
  const double* A;
  int64_t ld;
  b200_matvec_cb mv;
  void* user;
  b200_sparse_jac* sj;
  double shift;  // operator is A + shift I
  b200_mg* mg;   // LINOP_MULTIGRID: the hierarchy (owned when owns_mg)
  int32_t owns_mg;
  int64_t *csr_rowptr, *csr_col, *csr_map;  // LINOP_CSC: row view of the pattern (owned), built once so that y = A x is a deterministic gather
  b200_ilu0* ilu;  // LINOP_ILU0: the factors (borrowed)
  b200_amg* amg;   // LINOP_AMG: the hierarchy (borrowed)
};
enum { LINOP_PROBLEM = 0, LINOP_CSC = 1, LINOP_DENSE = 2, LINOP_CALLBACK = 3, LINOP_SPARSE_JAC = 4, LINOP_BLOCK_JACOBI = 5, LINOP_MULTIGRID = 6,
       LINOP_ILU0 = 7, LINOP_AMG = 8 };

// internal (non-ABI) helpers implemented across the .cu files
// Host callbacks run user device code on streams the library knows nothing about (its own stream is non-blocking): drain
// everything the library has enqueued before handing control to the callback.  The callback in turn must have finished its
// device work (or enqueued it on the context's stream) when it returns.
static inline int32_t b200i_sync_for_callback(b200_ctx* ctx) {
  if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) return B200_ERR_CUDA;
  if (ctx->aux_stream && cudaStreamSynchronize(ctx->aux_stream) != cudaSuccess) return B200_ERR_CUDA;
  return B200_OK;
}
int32_t b200i_linop_apply(b200_linop* op, const double* x, double* y);
// row view of a CSC pattern (ilu0.cu): int32 CSR with columns ascending, map = CSR position -> caller's CSC position, diag =
// the position of each row's diagonal (-1: none).  Empty string on success, else the message ("<who>: ..."; a missing
// diagonal, when required, names the row).
std::string b200i_csr_of_csc(const char* who, int64_t n, const int64_t* colptr, const int64_t* rowval, int32_t base, bool require_diag,
                             std::vector<int32_t>& rowptr, std::vector<int32_t>& col, std::vector<int32_t>& map, std::vector<int32_t>& diag);
// geometric multigrid preconditioner of the built-in Brusselator Jacobian (mg.cu)
int32_t b200i_mg_create(b200_problem* prob, b200_mg** out);
int32_t b200i_mg_destroy(b200_mg* mg);
int32_t b200i_mg_setup(b200_mg* mg, const double* u);   // rebuild the coarse operators for the linearisation point u
int32_t b200i_mg_apply(b200_mg* mg, const double* x, double* y);
int32_t b200i_mg_levels(b200_mg* mg, int32_t* nlev, int32_t* sizes, int32_t cap);
int32_t b200i_diag_shift(b200_ctx* ctx, int64_t n, double* A, int64_t ld, double shift);  // A[i,i] += shift
// column-pivoted Householder QR solve of a (possibly rank-deficient) dense system: the rescue of a singular LU
int32_t b200i_qrcp_solve(b200_ctx* ctx, int64_t n, double* A, int64_t ld, double* b, double* x, double* work, int32_t* jpvt_dev, int32_t* rank_host);
int32_t b200i_gram(b200_ctx* ctx, int64_t n, const double* J, int64_t ld, double* C, int64_t ldc);          // C = J' J
int32_t b200i_klement_descent(b200_ctx* ctx, int64_t n, const double* J, const double* fu, double* du);                       // du = -fu ./ J
int32_t b200i_klement_update(b200_ctx* ctx, int64_t n, double* J, const double* fu, double* fu_cache, const double* du);       // Klement's diagonal rule; fu_cache = fu
int32_t b200i_ger(b200_ctx* ctx, int64_t n, double* A, int64_t ld, const double* c, const double* w);              // A += c w'
int32_t b200i_scaled_identity(b200_ctx* ctx, int64_t n, double* A, int64_t ld, double d);                          // A = d I
int32_t b200i_lm_damp(b200_ctx* ctx, int64_t n, double* C, int64_t ldc, double* dtd, double lambda);     // dtd = max(dtd, diag C); C += lambda diag(dtd)
void b200i_sparse_jac_csr(b200_sparse_jac* sj, const int64_t** rowptr, const int64_t** csr_col, const int64_t** csr_map);
int32_t b200i_residual_norm(b200_problem* prob, const double* u, double* du, double* d_norminf /*device, pre-zeroed*/);
int32_t b200i_axpy_norm(b200_ctx* ctx, int64_t n, double a, const double* x, double* y, double* d_sumsq /*device, pre-zeroed*/);
int32_t b200i_reduce_sum_dev(b200_ctx* ctx, int64_t n, const double* x, const double* y, int mode, double* d_out, double a = 0.0);
int32_t b200i_fetch_scalars(b200_ctx* ctx, int count);  // d_scalars[0..count) -> h_scalars, synchronises
